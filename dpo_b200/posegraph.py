"""Host-side pose-graph utilities of the product: the data formats on either side of the hot path.

One-shot setup work (reader, Laplacian block assembly, initial guess), kept on the host as in the
reference (src/DPGO_utils.cpp).  Nothing here runs per iteration; the per-iteration path is the
CUDA library.  Function names follow the reference's DPGO_utils.h.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import numpy as np


@dataclass
class RelativeSEMeasurement:
    """ref: include/DPGO/RelativeSEMeasurement.h:21-50."""
    r1: int
    r2: int
    p1: int
    p2: int
    R: np.ndarray
    t: np.ndarray
    kappa: float
    tau: float
    isKnownInlier: bool = False
    weight: float = 1.0


class EdgeSet:
    """Struct-of-arrays container for a batch of RelativeSEMeasurement (what the kernels consume)."""

    def __init__(self, d: int, r1, r2, p1, p2, R, t, kappa, tau, weight=None):
        m = len(p1)
        self.d = d
        self.r1 = np.asarray(r1, dtype=np.int64).reshape(m)
        self.r2 = np.asarray(r2, dtype=np.int64).reshape(m)
        self.p1 = np.asarray(p1, dtype=np.int64).reshape(m)
        self.p2 = np.asarray(p2, dtype=np.int64).reshape(m)
        self.R = np.asarray(R, dtype=np.float64).reshape(m, d, d)
        self.t = np.asarray(t, dtype=np.float64).reshape(m, d)
        self.kappa = np.asarray(kappa, dtype=np.float64).reshape(m)
        self.tau = np.asarray(tau, dtype=np.float64).reshape(m)
        self.weight = np.ones(m) if weight is None else np.asarray(weight, dtype=np.float64).reshape(m)

    def __len__(self):
        return self.p1.shape[0]

    def take(self, idx) -> "EdgeSet":
        idx = np.asarray(idx, dtype=np.int64)
        return EdgeSet(self.d, self.r1[idx], self.r2[idx], self.p1[idx], self.p2[idx], self.R[idx], self.t[idx],
                       self.kappa[idx], self.tau[idx], self.weight[idx])

    @staticmethod
    def empty(d: int) -> "EdgeSet":
        return EdgeSet(d, [], [], [], [], np.zeros((0, d, d)), np.zeros((0, d)), [], [])

    @staticmethod
    def join(parts: Sequence["EdgeSet"]) -> "EdgeSet":
        d = parts[0].d
        c = lambda k: np.concatenate([getattr(p, k) for p in parts])
        return EdgeSet(d, c("r1"), c("r2"), c("p1"), c("p2"), c("R"), c("t"), c("kappa"), c("tau"), c("weight"))

    def to_list(self) -> List[RelativeSEMeasurement]:
        return [RelativeSEMeasurement(int(self.r1[k]), int(self.r2[k]), int(self.p1[k]), int(self.p2[k]),
                                      self.R[k].copy(), self.t[k].copy(), float(self.kappa[k]), float(self.tau[k]),
                                      False, float(self.weight[k])) for k in range(len(self))]

    def homogeneous(self) -> np.ndarray:
        """(m, d+1, d+1) matrices [R t; 0 1]."""
        m, d = len(self), self.d
        T = np.zeros((m, d + 1, d + 1))
        T[:, :d, :d] = self.R
        T[:, :d, d] = self.t
        T[:, d, d] = 1.0
        return T

    def omega(self) -> np.ndarray:
        """(m, d+1) diagonal weights (kappa..kappa, tau) * weight."""
        m, d = len(self), self.d
        om = np.empty((m, d + 1))
        om[:, :d] = (self.weight * self.kappa)[:, None]
        om[:, d] = self.weight * self.tau
        return om


def _inv_trace(sym: np.ndarray) -> float:
    return float(np.trace(np.linalg.inv(sym)))


def read_g2o_file(filename: str) -> Tuple[EdgeSet, int]:
    """Parse EDGE_SE2 / EDGE_SE3:QUAT records.  ref: read_g2o_file, src/DPGO_utils.cpp:64-197.

    kappa/tau are the information-divergence-minimising isotropic precisions (:121-125, :166-175);
    the quaternion is converted WITHOUT normalisation, as Eigen's toRotationMatrix does (:160).
    """
    p1, p2, Rs, ts, kap, tau = [], [], [], [], [], []
    d = 0
    with open(filename, "r") as fh:
        for line in fh:
            if line.startswith("EDGE_SE3:QUAT"):
                f = line.split()
                i, j = int(f[1]), int(f[2])
                x = [float(s) for s in f[3:31]]
                qx, qy, qz, qw = x[3], x[4], x[5], x[6]
                info = np.zeros((6, 6))
                info[np.triu_indices(6)] = x[7:28]
                info = info + np.triu(info, 1).T
                s2 = 2.0
                R = np.array([
                    [1 - s2 * (qy * qy + qz * qz), s2 * (qx * qy - qw * qz), s2 * (qx * qz + qw * qy)],
                    [s2 * (qx * qy + qw * qz), 1 - s2 * (qx * qx + qz * qz), s2 * (qy * qz - qw * qx)],
                    [s2 * (qx * qz - qw * qy), s2 * (qy * qz + qw * qx), 1 - s2 * (qx * qx + qy * qy)]])
                d = 3
                Rs.append(R)
                ts.append(x[0:3])
                tau.append(3.0 / _inv_trace(info[:3, :3]))
                kap.append(3.0 / (2.0 * _inv_trace(info[3:, 3:])))
            elif line.startswith("EDGE_SE2"):
                f = line.split()
                i, j = int(f[1]), int(f[2])
                dx, dy, th, I11, I12, I13, I22, I23, I33 = (float(s) for s in f[3:12])
                d = 2
                Rs.append(np.array([[math.cos(th), -math.sin(th)], [math.sin(th), math.cos(th)]]))
                ts.append([dx, dy])
                tau.append(2.0 / _inv_trace(np.array([[I11, I12], [I12, I22]])))
                kap.append(I33)
            elif line.startswith("VERTEX_SE") or not line.strip():
                continue
            else:
                raise ValueError("Error: unrecognized type: " + line.split()[0] + "!")
            p1.append(i)
            p2.append(j)
    m = len(p1)
    num_poses = (max(max(p1), max(p2)) + 1) if m else 1
    z = np.zeros(m, dtype=np.int64)
    return EdgeSet(d, z, z.copy(), p1, p2, np.array(Rs).reshape(m, d, d), np.array(ts).reshape(m, d), kap, tau), num_poses


def connection_laplacian_blocks(edges: EdgeSet):
    """Block triplets of Q = A Omega A^T.  ref: constructConnectionLaplacianSE, src/DPGO_utils.cpp:199-271.

    Per edge i->j:  Q_ii += T Om T^T,  Q_jj += Om,  Q_ij = -T Om,  Q_ji = -Om T^T.
    Returns (brow, bcol, blocks) with duplicates NOT merged (the library sums them).
    """
    m, dh = len(edges), edges.d + 1
    T = edges.homogeneous()
    om = edges.omega()
    TOm = T * om[:, None, :]
    blocks = np.empty((4 * m, dh, dh))
    blocks[0:m] = TOm @ np.transpose(T, (0, 2, 1))
    blocks[m:2 * m] = 0.0
    ar = np.arange(dh)
    blocks[m:2 * m, ar, ar] = om
    blocks[2 * m:3 * m] = -TOm
    blocks[3 * m:4 * m] = -np.transpose(TOm, (0, 2, 1))
    brow = np.concatenate([edges.p1, edges.p2, edges.p1, edges.p2]).astype(np.int32)
    bcol = np.concatenate([edges.p1, edges.p2, edges.p2, edges.p1]).astype(np.int32)
    return brow, bcol, blocks


def constructConnectionLaplacianSE(edges: EdgeSet, n: Optional[int] = None):
    """Scalar CSR (scipy) form, for callers that want the reference's SparseMatrix."""
    import scipy.sparse as sp
    dh = edges.d + 1
    if n is None:
        n = int(max(edges.p1.max(), edges.p2.max())) + 1
    brow, bcol, blocks = connection_laplacian_blocks(edges)
    bsr = sp.coo_matrix((np.ones(len(brow)), (brow, bcol)), shape=(n, n))   # structure only
    del bsr
    k, c = np.meshgrid(np.arange(dh), np.arange(dh), indexing="ij")
    rows = (brow[:, None, None].astype(np.int64) * dh + k[None]).ravel()
    cols = (bcol[:, None, None].astype(np.int64) * dh + c[None]).ravel()
    Q = sp.coo_matrix((blocks.ravel(), (rows, cols)), shape=(n * dh, n * dh)).tocsr()
    Q.sum_duplicates()
    return Q


def projectToRotationGroup(M: np.ndarray) -> np.ndarray:
    """ref: src/DPGO_utils.cpp:463-477."""
    U, _, Vt = np.linalg.svd(M)
    if np.linalg.det(U) * np.linalg.det(Vt) <= 0:
        U = U.copy()
        U[:, -1] = -U[:, -1]
    return U @ Vt


def fixedStiefelVariable(d: int, r: int) -> np.ndarray:
    """Deterministic element of St(d, r) shared by all agents as the lifting matrix.

    ref: src/DPGO_utils.cpp:487-492 (ROPTLIB RandInManifold after srand(1): value unpinned, any
    orthonormal r x d matrix is equivalent -- cost and gradient norm are invariant under it).
    """
    M = np.zeros((r, d))
    rng = np.random.RandomState(1)
    M[:] = rng.standard_normal((r, d))
    Qm, Rm = np.linalg.qr(M)
    return Qm * np.sign(np.diag(Rm))[None, :]


def odometryInitialization(d: int, n: int, odometry: EdgeSet) -> np.ndarray:
    """ref: src/DPGO_utils.cpp:411-432."""
    T = np.zeros((d, (d + 1) * n))
    R = np.eye(d)
    t = np.zeros(d)
    T[:, :d] = R
    for k in range(len(odometry)):
        assert odometry.p1[k] == k and odometry.p2[k] == k + 1
        t = t + R @ odometry.t[k]
        R = R @ odometry.R[k]
        T[:, (k + 1) * (d + 1):(k + 1) * (d + 1) + d] = R
        T[:, (k + 1) * (d + 1) + d] = t
    return T


def chordalInitialization(d: int, n: int, edges: EdgeSet) -> np.ndarray:
    """Chordal relaxation: rotations by linear least squares + projection, then translations.

    ref: chordalInitialization / recoverTranslations, src/DPGO_utils.cpp:362-409, 434-461 (two sparse
    least-squares problems, SPQR there; sparse normal equations + refinement here).  Pose 0 is the
    gauge: R_0 = I, t_0 = 0.
    """
    import scipy.sparse as sp
    import scipy.sparse.linalg as spla
    m = len(edges)
    i, j = edges.p1, edges.p2
    sk, st = np.sqrt(edges.kappa), np.sqrt(edges.tau)

    def solve_ls(A, b):
        A = A.tocsc()
        lu = spla.splu((A.T @ A).tocsc())
        x = lu.solve(A.T @ b)
        for _ in range(2):
            x += lu.solve(A.T @ (b - A @ x))
        return x

    # rotations: minimise sum_e kappa_e |R_j - R_i Rij|_F^2 over unconstrained d x d blocks, R_0 = I.
    # Unknown vec(R_p) column-major (entry (l, c) at d*c + l).  Row (e, r, l):  R_j[l, r] - sum_c R_i[l, c] Rij[c, r]
    d2 = d * d
    e_idx = np.arange(m)
    rr, cc, ll = np.meshgrid(np.arange(d), np.arange(d), np.arange(d), indexing="ij")
    rows_a = (e_idx[:, None, None, None] * d2 + rr[None] * d + ll[None]).ravel()
    cols_a = (i[:, None, None, None] * d2 + cc[None] * d + ll[None]).ravel()
    vals_a = (-sk[:, None, None, None] * np.transpose(edges.R, (0, 2, 1))[:, :, :, None] * np.ones((1, 1, 1, d))).ravel()
    rl = np.arange(d2)
    rows_b = (e_idx[:, None] * d2 + rl[None]).ravel()
    cols_b = (j[:, None] * d2 + rl[None]).ravel()
    vals_b = np.repeat(sk, d2)
    A = sp.coo_matrix((np.concatenate([vals_a, vals_b]), (np.concatenate([rows_a, rows_b]),
                                                          np.concatenate([cols_a, cols_b]))),
                      shape=(d2 * m, d2 * n)).tocsc()
    rhs = -(A[:, :d2] @ np.eye(d).reshape(-1, order="F"))
    sol = solve_ls(A[:, d2:], rhs)
    Rall = np.zeros((n, d, d))
    Rall[0] = np.eye(d)
    Rall[1:] = np.transpose(sol.reshape(n - 1, d, d), (0, 2, 1))       # column-major vec -> matrix
    for p in range(1, n):
        Rall[p] = projectToRotationGroup(Rall[p])
    # translations: minimise sum_e tau_e |t_j - t_i - R_i tij|^2, t_0 = 0
    l = np.arange(d)
    rows = (e_idx[:, None] * d + l[None]).ravel()
    B = sp.coo_matrix((np.concatenate([np.repeat(-st, d), np.repeat(st, d)]),
                       (np.concatenate([rows, rows]),
                        np.concatenate([(i[:, None] * d + l[None]).ravel(), (j[:, None] * d + l[None]).ravel()]))),
                      shape=(d * m, d * n)).tocsc()
    c = (st[:, None] * np.einsum("mab,mb->ma", Rall[i], edges.t)).ravel()
    tsol = solve_ls(B[:, d:], c)
    T = np.zeros((d, (d + 1) * n))
    tt = np.zeros((n, d))
    tt[1:] = tsol.reshape(n - 1, d)
    for p in range(n):
        T[:, p * (d + 1):p * (d + 1) + d] = Rall[p]
        T[:, p * (d + 1) + d] = tt[p]
    return T


def chordalInitializationGPU(d: int, n: int, edges: EdgeSet, device: int = 0, tol: float = 1e-11, max_iter: int = 50000,
                             return_iterations: bool = False):
    """chordalInitialization on the GPU (dpgo_chordal_initialization): both least-squares problems by Jacobi-preconditioned
    conjugate gradients over the hot path's block-CSR product kernel.  ref src/DPGO_utils.cpp:273-461."""
    import ctypes as C
    from . import _capi as capi
    lib = capi.load_library()
    p1 = np.ascontiguousarray(edges.p1, dtype=np.int32)
    p2 = np.ascontiguousarray(edges.p2, dtype=np.int32)
    R = np.ascontiguousarray(edges.R, dtype=np.float64)
    t = np.ascontiguousarray(edges.t, dtype=np.float64)
    kappa = np.ascontiguousarray(edges.kappa * edges.weight, dtype=np.float64)
    tau = np.ascontiguousarray(edges.tau * edges.weight, dtype=np.float64)
    T = np.zeros((d, (d + 1) * n), order="F")
    its = (C.c_int32 * 2)()
    code = lib.dpgo_chordal_initialization(n, d, len(p1), capi.iptr(p1), capi.iptr(p2), capi.dptr(R), capi.dptr(t), capi.dptr(kappa),
                                           capi.dptr(tau), device, tol, max_iter, capi.dptr(T), its)
    if code != capi.OK:
        raise capi.DpgoError(code, lib.dpgo_chordal_last_error().decode("utf-8", "replace"))
    return (T, (int(its[0]), int(its[1]))) if return_iterations else T


def _covariance_args(edges: EdgeSet, n: int, T: np.ndarray, pairs):
    d = edges.d
    T = np.asfortranarray(np.asarray(T, dtype=np.float64))
    if T.shape != (d, (d + 1) * n):
        raise ValueError(f"expected a trajectory of shape {(d, (d + 1) * n)}, got {T.shape}")
    pr = np.zeros((0, 2), dtype=np.int32) if pairs is None else np.ascontiguousarray(np.asarray(pairs, dtype=np.int32).reshape(-1, 2))
    arrays = [np.ascontiguousarray(a, dtype=dt) for a, dt in ((edges.p1, np.int32), (edges.p2, np.int32), (edges.R, np.float64),
                                                            (edges.t, np.float64), (edges.kappa, np.float64),
                                                            (edges.tau, np.float64), (edges.weight, np.float64))]
    b = 6 if d == 3 else 3
    return T, pr, arrays, b


def poseCovariancesGPU(edges: EdgeSet, n: int, T: np.ndarray, anchor: int = 0, pairs=None, device: int = 0,
                       return_info: bool = False):
    """Marginal covariances of the poses of trajectory T (d x (d+1)n, e.g. a rounded solution) under the Gauss-Newton
    information of `edges`, with pose `anchor` fixed (dpgo_pose_covariances; the model is in include/dpgo_b200.h).

    Returns cov (n, b, b), b = 6 (SE(3): rotation then translation) or 3 (SE(2): angle then translation), the anchor's
    block 0; with pairs (k, 2) also the cross blocks Sigma[x_i, x_j] (k, b, b); with return_info also info16.
    The graph is assembled, factored and selectively inverted on the GPU; edge weights are honoured."""
    import ctypes as C
    from . import _capi as capi
    lib = capi.load_library()
    T, pr, (p1, p2, R, t, kappa, tau, w), b = _covariance_args(edges, n, T, pairs)
    cov = np.zeros((n, b, b))
    pcov = np.zeros((max(len(pr), 1), b, b))
    info = (C.c_int64 * 16)()
    capi.check(lib.dpgo_pose_covariances(n, edges.d, len(p1), capi.iptr(p1), capi.iptr(p2), capi.dptr(R), capi.dptr(t),
                                         capi.dptr(kappa), capi.dptr(tau), capi.dptr(w), capi.dptr(T), int(anchor), device,
                                         len(pr), capi.iptr(pr), capi.dptr(cov), capi.dptr(pcov), info))
    out = (cov,) if pairs is None else (cov, pcov[:len(pr)])
    if return_info:
        out = out + (list(info),)
    return out[0] if len(out) == 1 else out


def synthetic_grid_graph(nx: int, ny: int, nz: int, edges_per_pose: float = 4.0, seed: int = 0,
                         rot_sigma: float = 0.05, trans_sigma: float = 0.1, kappa: float = 200.0,
                         tau: float = 100.0) -> Tuple[EdgeSet, int, np.ndarray]:
    """SURVEY 8(d) config 5: poses on an nx x ny x nz lattice numbered along a boustrophedon path
    (consecutive ids are lattice neighbours -> odometry chain), all remaining lattice-neighbour pairs
    as loop closures, plus seeded random closures between poses at lattice distance <= 3 until
    edges_per_pose * n unique edges.  Returns (edges, n, ground-truth T of shape (3, 4n))."""
    rng = np.random.default_rng(seed)
    n = nx * ny * nz
    ids = -np.ones((nx, ny, nz), dtype=np.int64)
    coords = np.zeros((n, 3), dtype=np.int64)
    k = 0
    row = 0
    for z in range(nz):
        ys = range(ny) if z % 2 == 0 else range(ny - 1, -1, -1)
        for y in ys:
            xs = np.arange(nx) if row % 2 == 0 else np.arange(nx - 1, -1, -1)
            ids[xs, y, z] = k + np.arange(nx)
            coords[k:k + nx, 0] = xs
            coords[k:k + nx, 1] = y
            coords[k:k + nx, 2] = z
            k += nx
            row += 1
    enc = []
    for ax, shape in ((0, nx), (1, ny), (2, nz)):
        sl_a = [slice(None)] * 3
        sl_b = [slice(None)] * 3
        sl_a[ax] = slice(0, shape - 1)
        sl_b[ax] = slice(1, shape)
        a, b = ids[tuple(sl_a)].ravel(), ids[tuple(sl_b)].ravel()
        enc.append(np.minimum(a, b) * n + np.maximum(a, b))
    chain = np.arange(n - 1, dtype=np.int64)
    enc.append(chain * n + chain + 1)                 # boustrophedon chain (lattice neighbours by construction)
    keys = np.unique(np.concatenate(enc))
    target = int(round(edges_per_pose * n))
    dims = np.array([nx, ny, nz])
    while keys.shape[0] < target:
        need = target - keys.shape[0]
        src = rng.integers(0, n, size=2 * need + 16)
        dst_c = coords[src] + rng.integers(-3, 4, size=(src.shape[0], 3))
        ok = ((dst_c >= 0) & (dst_c < dims)).all(axis=1)
        src, dst_c = src[ok], dst_c[ok]
        dst = ids[dst_c[:, 0], dst_c[:, 1], dst_c[:, 2]]
        ok = dst != src
        cand = np.minimum(src[ok], dst[ok]) * n + np.maximum(src[ok], dst[ok])
        _, first = np.unique(cand, return_index=True)
        cand = cand[np.sort(first)]                   # first occurrences, draw order preserved
        cand = cand[~np.isin(cand, keys)][:need]
        keys = np.unique(np.concatenate([keys, cand]))
    p1, p2 = keys // n, keys % n
    m = keys.shape[0]
    # ground truth: lattice positions, random rotations (normalised 4-vector of N(0,1))
    q = rng.standard_normal((n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    Rgt = np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
                    np.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
                    np.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)], 1)
    tgt = coords.astype(np.float64)
    Rrel = np.einsum("mba,mbc->mac", Rgt[p1], Rgt[p2])
    trel = np.einsum("mba,mb->ma", Rgt[p1], tgt[p2] - tgt[p1])
    aa = rot_sigma * rng.standard_normal((m, 3))
    ang = np.linalg.norm(aa, axis=1)
    ax_ = aa / np.maximum(ang, 1e-300)[:, None]
    K = np.zeros((m, 3, 3))
    K[:, 0, 1], K[:, 0, 2], K[:, 1, 0] = -ax_[:, 2], ax_[:, 1], ax_[:, 2]
    K[:, 1, 2], K[:, 2, 0], K[:, 2, 1] = -ax_[:, 0], -ax_[:, 1], ax_[:, 0]
    Rn = np.eye(3)[None] + np.sin(ang)[:, None, None] * K + (1 - np.cos(ang))[:, None, None] * (K @ K)
    Rmeas = Rrel @ Rn
    tmeas = trel + trans_sigma * rng.standard_normal((m, 3))
    zz = np.zeros(m, dtype=np.int64)
    edges = EdgeSet(3, zz, zz.copy(), p1, p2, Rmeas, tmeas, np.full(m, kappa), np.full(m, tau))
    Tgt = np.zeros((3, 4 * n))
    Tgt.reshape(3, n, 4)[:, :, :3] = np.transpose(Rgt, (1, 0, 2))
    Tgt.reshape(3, n, 4)[:, :, 3] = tgt.T
    return edges, n, Tgt


def grid_lattice_coords(nx: int, ny: int, nz: int) -> np.ndarray:
    """(n, 3) lattice coordinates of the poses of synthetic_grid_graph (ids follow the boustrophedon path)."""
    n = nx * ny * nz
    coords = np.zeros((n, 3), dtype=np.int64)
    k = 0
    row = 0
    for z in range(nz):
        ys = range(ny) if z % 2 == 0 else range(ny - 1, -1, -1)
        for y in ys:
            xs = np.arange(nx) if row % 2 == 0 else np.arange(nx - 1, -1, -1)
            coords[k:k + nx, 0] = xs
            coords[k:k + nx, 1] = y
            coords[k:k + nx, 2] = z
            k += nx
            row += 1
    return coords


def grid_block_owner(nx: int, ny: int, nz: int, k: int) -> np.ndarray:
    """Pose -> agent for the synthetic lattice: k = kx*ky*kz rectangular blocks with the smallest total cut surface
    (BASELINE config 5 with 8 agents: 2 x 2 x 2 blocks).  The contiguous id ranges of examples/MultiRobotExample.cpp:95-109
    cut a 100 x 100 x 10 lattice into 1.25-layer slabs in which EVERY pose is public; blocks keep the public poses at the
    block faces.  Use as DistributedPGO(..., owner=grid_block_owner(...))."""
    best = None
    for kx in range(1, k + 1):
        if k % kx:
            continue
        for ky in range(1, k // kx + 1):
            if (k // kx) % ky:
                continue
            kz = k // (kx * ky)
            if kx > nx or ky > ny or kz > nz:
                continue
            cut = (kx - 1) * ny * nz + (ky - 1) * nx * nz + (kz - 1) * nx * ny
            if best is None or cut < best[0]:
                best = (cut, kx, ky, kz)
    if best is None:
        raise ValueError(f"cannot cut a {nx}x{ny}x{nz} lattice into {k} blocks")
    _, kx, ky, kz = best
    c = grid_lattice_coords(nx, ny, nz)
    bx = np.minimum(c[:, 0] * kx // nx, kx - 1)
    by = np.minimum(c[:, 1] * ky // ny, ky - 1)
    bz = np.minimum(c[:, 2] * kz // nz, kz - 1)
    return ((bz * ky + by) * kx + bx).astype(np.int64)


def read_partition_file(path: str, n: int | None = None) -> np.ndarray:
    """Pose -> agent map from a graph-partition file, one agent id per line in pose order
    (ref examples/MultiRobotExample.cpp:76-91: graph/<robots>/<strength>/<dataset>)."""
    owner = np.loadtxt(path, dtype=np.int64, ndmin=1)
    if n is not None and owner.shape[0] != n:
        raise ValueError(f"partition file has {owner.shape[0]} lines, the pose graph has {n} poses")
    if owner.min() < 0:
        raise ValueError("negative agent id in the partition file")
    return owner


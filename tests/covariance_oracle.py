"""NumPy / SciPy restatement of the pose-covariance model of dpgo_pose_covariances (include/dpgo_b200.h).

Right perturbations R_i exp([w_i]x), t_i + R_i v_i with tangent x_i = (w_i, v_i) (b = 6 in 3D, 3 in 2D); per edge
i -> j the residuals r_rot = R_j - R_i Rt (weight kappa, row-major) and r_tra = t_j - t_i - R_i tt (weight tau), so that
sum_e 1/2 r^T Om r equals f = 1/2 <Q, T^T T>; H = sum_e J^T Om J (Gauss-Newton) and Sigma = H_anchored^-1.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla


def tangent_dim(d: int) -> int:
    return 6 if d == 3 else 3


def generators(d: int) -> np.ndarray:
    if d == 2:
        return np.array([[[0.0, -1.0], [1.0, 0.0]]])
    G = np.zeros((3, 3, 3))
    for k in range(3):
        a, c = (k + 1) % 3, (k + 2) % 3
        G[k, a, c], G[k, c, a] = -1.0, 1.0
    return G


def exp_so(d: int, w) -> np.ndarray:
    w = np.atleast_1d(np.asarray(w, dtype=np.float64))
    K = np.einsum("k,kab->ab", w, generators(d))
    if d == 2:
        c, s = np.cos(w[0]), np.sin(w[0])
        return np.array([[c, -s], [s, c]])
    th = np.linalg.norm(w)
    if th < 1e-12:
        return np.eye(3) + K
    return np.eye(3) + np.sin(th) / th * K + (1 - np.cos(th)) / th ** 2 * (K @ K)


def poses(T: np.ndarray, d: int):
    n = T.shape[1] // (d + 1)
    Tp = T.reshape(d, n, d + 1).transpose(1, 0, 2)
    return Tp[:, :, :d], Tp[:, :, d]


def residuals(T, edges):
    """(m, d*d + d) residuals and (m, d*d + d) diagonal weights."""
    d = edges.d
    R, t = poses(T, d)
    i, j = edges.p1, edges.p2
    rr = (R[j] - R[i] @ edges.R).reshape(len(edges), d * d)
    rt = t[j] - t[i] - np.einsum("mab,mb->ma", R[i], edges.t)
    om = np.concatenate([np.repeat((edges.weight * edges.kappa)[:, None], d * d, 1),
                         np.repeat((edges.weight * edges.tau)[:, None], d, 1)], axis=1)
    return np.concatenate([rr, rt], axis=1), om


def jacobians(T, edges):
    """(m, d*d + d, b) Jacobians of each edge's residual with respect to x_i and x_j."""
    d = edges.d
    b, nw = tangent_dim(d), (3 if d == 3 else 1)
    R, _ = poses(T, d)
    i, j = edges.p1, edges.p2
    m = len(edges)
    dt = np.result_type(T, edges.R)                      # long double in, long double Jacobians out
    Ji, Jj = np.zeros((m, d * d + d, b), dtype=dt), np.zeros((m, d * d + d, b), dtype=dt)
    for k, G in enumerate(generators(d)):
        Jj[:, :d * d, k] = (R[j] @ G).reshape(m, d * d)
        RG = R[i] @ G
        Ji[:, :d * d, k] = -(RG @ edges.R).reshape(m, d * d)
        Ji[:, d * d:, k] = -np.einsum("mab,mb->ma", RG, edges.t)
    for k in range(d):
        Jj[:, d * d:, nw + k] = R[j][:, :, k]
        Ji[:, d * d:, nw + k] = -R[i][:, :, k]
    return Ji, Jj


def information(T, edges, n: int) -> sp.csr_matrix:
    """Gauss-Newton information H (n b x n b), no anchoring."""
    d = edges.d
    b = tangent_dim(d)
    Ji, Jj = jacobians(T, edges)
    _, om = residuals(T, edges)
    rows, cols, vals = [], [], []
    idx = np.arange(b)
    for (A, pa) in ((Ji, edges.p1), (Jj, edges.p2)):
        for (B, pc) in ((Ji, edges.p1), (Jj, edges.p2)):
            blk = np.einsum("mra,mr,mrc->mac", A, om, B)
            rows.append((pa[:, None, None] * b + idx[None, :, None] + 0 * idx[None, None, :]).ravel())
            cols.append((pc[:, None, None] * b + idx[None, None, :] + 0 * idx[None, :, None]).ravel())
            vals.append(blk.ravel())
    H = sp.coo_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(n * b, n * b)).tocsr()
    H.sum_duplicates()
    return H


def free_index(n: int, b: int, anchor: int) -> np.ndarray:
    keep = np.ones(n * b, dtype=bool)
    keep[anchor * b:(anchor + 1) * b] = False
    return np.nonzero(keep)[0]


def covariances_dense(H, n: int, b: int, anchor: int = 0) -> np.ndarray:
    """Full Sigma (n b x n b, anchor rows / columns zero) by a dense inverse (small graphs)."""
    f = free_index(n, b, anchor)
    S = np.zeros((n * b, n * b))
    S[np.ix_(f, f)] = np.linalg.inv(H[f][:, f].toarray())
    return S


def blocks_of(S, b: int, pairs):
    return np.stack([S[i * b:(i + 1) * b, j * b:(j + 1) * b] for i, j in pairs])


def covariance_columns(H, n: int, b: int, anchor: int, cols_of):
    """Sigma[:, x_p] for each pose p in cols_of by splu column solves: dict p -> (n b x b)."""
    return _columns(spla.splu(H[free_index(n, b, anchor)][:, free_index(n, b, anchor)].tocsc()), n, b, anchor, cols_of)


def _columns(lu, n, b, anchor, cols_of):
    f = free_index(n, b, anchor)
    free = [int(p) for p in cols_of if p != anchor]
    E = np.zeros((len(f), b * len(free)))
    for q, p in enumerate(free):
        E[np.searchsorted(f, np.arange(p * b, (p + 1) * b)), q * b + np.arange(b)] = 1.0
    Xf = lu.solve(E) if free else E
    out = {}
    for p in cols_of:
        X = np.zeros((n * b, b))
        if p != anchor:
            q = free.index(int(p))
            X[f] = Xf[:, q * b:(q + 1) * b]
        out[int(p)] = X
    return out


def refine(lu, A, E, X, steps: int = 2):
    """Iterative refinement of the solves X ~ A^-1 E with the residual E - A X in extended precision (np.longdouble):
    the forward error then no longer carries splu's cond(A) eps, which matters on ill-conditioned graphs.  A is a SciPy
    sparse matrix, or a function returning the long-double product A X of a long-double block of columns X: for a
    matrix whose values are themselves long double, so that the residuals come from those values rather than from the
    doubles lu factored."""
    if callable(A):
        product = A
    else:
        A = A.tocsr()
        data, idx, ptr = A.data.astype(np.longdouble), A.indices, A.indptr
        assert np.all(np.diff(ptr) > 0)
        product = lambda Xc: np.add.reduceat(data[:, None] * Xc[idx], ptr[:-1], axis=0)
    Xl = X.astype(np.longdouble)
    for _ in range(steps):
        Rs = np.empty(X.shape)
        for c0 in range(0, X.shape[1], 16):
            c1 = min(X.shape[1], c0 + 16)
            AX = product(Xl[:, c0:c1])
            Rs[:, c0:c1] = (E[:, c0:c1].astype(np.longdouble) - AX).astype(np.float64)
        Xl += lu.solve(Rs).astype(np.longdouble)
    return Xl.astype(np.float64)


def block_sample(H, n: int, b: int, anchor: int, pairs, batch: int = 100):
    """Sigma blocks [x_i, x_j] for (i, j) in pairs by refined splu column solves over the distinct j, `batch` poses at a
    time."""
    pairs = [(int(i), int(j)) for i, j in pairs]
    f = free_index(n, b, anchor)
    Hf = H[f][:, f].tocsc()
    lu = spla.splu(Hf)
    out = {}
    cols = sorted({j for _, j in pairs if j != anchor})
    for k in range(0, len(cols), batch):
        part = cols[k:k + batch]
        E = np.zeros((len(f), b * len(part)))
        for q, p in enumerate(part):
            E[np.searchsorted(f, np.arange(p * b, (p + 1) * b)), q * b + np.arange(b)] = 1.0
        Xf = refine(lu, Hf, E, lu.solve(E))
        for q, p in enumerate(part):
            X = np.zeros((n * b, b))
            X[f] = Xf[:, q * b:(q + 1) * b]
            for i, j in pairs:
                if j == p:
                    out[(i, j)] = X[i * b:(i + 1) * b]
    return np.stack([out.get(p, np.zeros((b, b))) for p in pairs])


def perturb(T, d: int, p: int, x) -> np.ndarray:
    """T with pose p moved by the right perturbation x = (w, v)."""
    nw = 3 if d == 3 else 1
    T = T.copy()
    c0 = p * (d + 1)
    R = T[:, c0:c0 + d].copy()
    T[:, c0:c0 + d] = R @ exp_so(d, x[:nw])
    T[:, c0 + d] = T[:, c0 + d] + R @ np.asarray(x[nw:])
    return T


def random_trajectory(d: int, n: int, rng) -> np.ndarray:
    T = np.zeros((d, (d + 1) * n))
    for p in range(n):
        w = rng.standard_normal(3 if d == 3 else 1)
        T[:, p * (d + 1):p * (d + 1) + d] = exp_so(d, w)
        T[:, p * (d + 1) + d] = rng.standard_normal(d) * 3.0
    return T


def edge_arrays(edges):
    """The C ABI's edge arrays (int32 endpoints, row-major R, t)."""
    return (np.ascontiguousarray(edges.p1, dtype=np.int32), np.ascontiguousarray(edges.p2, dtype=np.int32),
            np.ascontiguousarray(edges.R, dtype=np.float64), np.ascontiguousarray(edges.t, dtype=np.float64),
            np.ascontiguousarray(edges.kappa, dtype=np.float64), np.ascontiguousarray(edges.tau, dtype=np.float64),
            np.ascontiguousarray(edges.weight, dtype=np.float64))

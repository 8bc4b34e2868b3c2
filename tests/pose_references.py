"""40-digit references (mpmath) of the per-pose kernels: polar factor, projection onto SO(d) and QF retraction, and the
crafted tiles they are checked on.  Helper module of test_structure_cases.py (CPU) and test_gpu_pose_numerics.py (GPU)."""
from __future__ import annotations

import mpmath as mpm
import numpy as np

DPS = 40


def _mat(M):
    return mpm.matrix([[mpm.mpf(float(x)) for x in row] for row in np.asarray(M)])


def _np(A):
    return np.array([[float(A[i, j]) for j in range(A.cols)] for i in range(A.rows)])


def svd(M):
    """U (r x d), singular values (d), V (d x d) of an r x d matrix, r >= d, at DPS digits."""
    with mpm.workdps(DPS):
        U, S, V = mpm.svd_r(_mat(M), full_matrices=False)      # M = U diag(S) V  (V is V^T)
        return _np(U), np.array([float(s) for s in S]), _np(V).T


def polar(M):
    """U V^T of the thin SVD (the reference's projectToStiefelManifold), rounded from DPS digits."""
    with mpm.workdps(DPS):
        U, S, V = mpm.svd_r(_mat(M), full_matrices=False)
        return _np(U * V)


def rotation(M):
    """argmin_{R in SO(d)} |R - M|_F (the reference's projectToRotationGroup): U diag(1, .., det(U V^T)) V^T."""
    with mpm.workdps(DPS):
        U, S, V = mpm.svd_r(_mat(M))
        if mpm.det(U * V) < 0:
            U[:, U.cols - 1] = -U[:, U.cols - 1]
        return _np(U * V)


def qf(M):
    """Q factor of the thin QR with a positive diagonal of R (QF retraction), rounded from DPS digits."""
    with mpm.workdps(DPS):
        A = _mat(M)
        r, d = A.rows, A.cols
        Qm = mpm.matrix(r, d)
        for c in range(d):                       # modified Gram-Schmidt twice at DPS digits is exact enough
            v = A[:, c]
            for _ in range(2):
                for k in range(c):
                    h = sum(Qm[i, k] * v[i] for i in range(r))
                    v = v - h * Qm[:, k]
            nrm = mpm.sqrt(sum(v[i] ** 2 for i in range(r)))
            Qm[:, c] = v / nrm
        return _np(Qm)


def with_singular_values(rng, r, d, sig, det_sign=None):
    """r x d matrix U diag(sig) V^T with random orthonormal U, V; for r = d an optional determinant sign"""
    U = np.linalg.qr(rng.standard_normal((r, d)))[0]
    V = np.linalg.qr(rng.standard_normal((d, d)))[0]
    M = (U * np.asarray(sig, dtype=np.float64)[None, :]) @ V.T
    if det_sign is not None and np.sign(np.linalg.det(M)) != det_sign:
        M[:, 0] = -M[:, 0]
    return M


def crafted_tiles(rng, r, d):
    """(label, r x d matrix, polar factor unique?) for the inputs where an SVD-based projection goes wrong"""
    out = []
    spectra = {"ones": [1.0] * d, "graded": [1.0, 1e-4, 1e-8][:d], "wide": [1e3, 1.0, 1e-12][:d],
               "repeated": ([2.0, 2.0, 1e-3] if d == 3 else [2.0, 2.0])}
    for k, s in spectra.items():
        for rep in range(3):
            out.append((f"sv_{k}", with_singular_values(rng, r, d, s), True))
    for rep in range(3):
        out.append(("orthonormal", np.linalg.qr(rng.standard_normal((r, d)))[0], True))
    if r == d:
        for rep in range(4):
            out.append(("det_neg", with_singular_values(rng, r, d, rng.uniform(0.5, 2.0, d), det_sign=-1.0), True))
    for rep in range(2):
        M = rng.standard_normal((r, d))
        out.append(("scale_1e100", M * 1e100, True))
        out.append(("scale_1e-100", M * 1e-100, True))
    Z = rng.standard_normal((r, d))
    Z[:, -1] = 0.0
    out.append(("zero_column", Z, False))
    out.append(("rank_one", np.outer(rng.standard_normal(r), rng.standard_normal(d)), False))
    out.append(("all_zero", np.zeros((r, d)), False))
    return out

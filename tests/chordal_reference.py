"""High-precision CPU reference of the chordal initialisation, and the error bounds its GPU solver promises.  Helper module
of test_chordal_cpu.py (CPU) and test_gpu_chordal.py (GPU); no fixtures.

The two least-squares problems are built exactly as oracle.chordal_initialization builds them (the reference's B3 for the
rotations, B1 / B2 for the translations, gauge R_0 = I, t_0 = 0) and restricted to the connected component of pose 0 (the
poses joined to it by edges of positive weight), where their normal matrices are nonsingular.  Each is solved by a float64
sparse LU, refined with residuals taken in long double until the correction is far below any bound tested here.

Bounds.  dpgo_chordal_initialization stops its Jacobi-preconditioned CG when the recursive residual r satisfies
||D^-1/2 r|| <= tol ||D^-1/2 b|| (D = diag of the normal matrix A).  The true residual of the returned iterate differs from
the recursive one by rounding: at most c u (|| D^-1/2 |A| |x| || + || D^-1/2 |b| ||), c a small multiple of the longest row
(its dot length).  That residual bound, divided by lambda_min(D^-1/2 A D^-1/2), bounds the error in the D^1/2-norm, and
the projection onto SO(d) passes it on with the factor 2 / (sigma_{d-1} + sigma_d) of the unprojected matrix.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla
from scipy.sparse.csgraph import connected_components

LD = np.longdouble
U = 2.0 ** -53                       # unit roundoff of float64
DENSE_EIG_MAX = 1500                 # reduced systems up to this size get dense eigenvalues


class Coo:
    """A sparse float64 matrix as triplets, with products accumulated in long double (np.add.at)."""

    def __init__(self, rows, cols, vals, shape):
        self.rows = np.asarray(rows, dtype=np.int64)
        self.cols = np.asarray(cols, dtype=np.int64)
        self.vals = np.asarray(vals, dtype=np.float64)
        self.shape = shape

    def mul(self, x, absolute=False):
        """A x (A^T-free) in long double; absolute=True: |A| |x|"""
        v, x = (np.abs(self.vals), np.abs(np.asarray(x, dtype=LD))) if absolute else (self.vals, np.asarray(x, dtype=LD))
        y = np.zeros(self.shape[0], dtype=LD)
        np.add.at(y, self.rows, v.astype(LD) * x[self.cols])
        return y

    def tmul(self, y, absolute=False):
        """A^T y in long double; absolute=True: |A|^T |y|"""
        v, y = (np.abs(self.vals), np.abs(np.asarray(y, dtype=LD))) if absolute else (self.vals, np.asarray(y, dtype=LD))
        x = np.zeros(self.shape[1], dtype=LD)
        np.add.at(x, self.cols, v.astype(LD) * y[self.rows])
        return x

    def csc(self):
        return sp.coo_matrix((self.vals, (self.rows, self.cols)), shape=self.shape).tocsc()


# ---------------------------------------------------------------------------------------------------------------------
# the reference's least-squares matrices (same index conventions as oracle.chordal_initialization)
# ---------------------------------------------------------------------------------------------------------------------
def b3_matrix(edges, n) -> Coo:
    """B3 (d^2 m x d^2 n): row (e, r, l) = sqrt(kappa) (R_j[l, r] - sum_c R_i[l, c] R_ij[c, r]); unknown vec(R_p) column-major,
    entry (l, c) of R_p at p d^2 + d c + l.  R_ij is taken as given (no re-orthogonalisation)."""
    d, m = edges.d, len(edges)
    d2 = d * d
    e = np.arange(m)
    sqk = np.sqrt(edges.kappa)
    rr, cc, ll = np.meshgrid(np.arange(d), np.arange(d), np.arange(d), indexing="ij")
    rows_a = (e[:, None, None, None] * d2 + d * rr[None] + ll[None]).ravel()
    cols_a = (edges.p1[:, None, None, None] * d2 + d * cc[None] + ll[None]).ravel()
    vals_a = (-sqk[:, None, None, None] * np.transpose(edges.R, (0, 2, 1))[:, :, :, None] * np.ones((1, 1, 1, d))).ravel()
    l2 = np.arange(d2)
    rows_b = (e[:, None] * d2 + l2[None, :]).ravel()
    cols_b = (edges.p2[:, None] * d2 + l2[None, :]).ravel()
    return Coo(np.concatenate([rows_a, rows_b]), np.concatenate([cols_a, cols_b]),
               np.concatenate([vals_a, np.repeat(sqk, d2)]), (d2 * m, d2 * n))


def b1_matrix(edges, n) -> Coo:
    """B1 (d m x d n): row (e, l) = sqrt(tau) (t_j[l] - t_i[l]); unknown t_p[l] at p d + l."""
    d, m = edges.d, len(edges)
    e = np.arange(m)
    sqt = np.sqrt(edges.tau)
    l = np.arange(d)
    r = (e[:, None] * d + l[None, :]).ravel()
    return Coo(np.concatenate([r, r]),
               np.concatenate([(edges.p1[:, None] * d + l).ravel(), (edges.p2[:, None] * d + l).ravel()]),
               np.concatenate([np.repeat(-sqt, d), np.repeat(sqt, d)]), (d * m, d * n))


def b2_target(edges, R):
    """-B2 vec(R) of the reference: row (e, l) = sqrt(tau) (R_i t_ij)[l], in long double, and its absolute evaluation."""
    sqt = ld(np.sqrt(edges.tau))
    Ri, t = ld(np.asarray(R)[edges.p1]), ld(edges.t)
    val = sqt[:, None] * np.einsum("mab,mb->ma", Ri, t)
    mag = sqt[:, None] * np.einsum("mab,mb->ma", np.abs(Ri), np.abs(t))
    return val.ravel(), mag.ravel()


def ld(a):
    return np.asarray(a, dtype=LD)


def component_of_zero(n, p1, p2, w):
    """Boolean mask of the poses joined to pose 0 by edges of positive weight."""
    keep = np.asarray(w) > 0
    A = sp.coo_matrix((np.ones(int(keep.sum())), (np.asarray(p1)[keep], np.asarray(p2)[keep])), shape=(n, n))
    _, lab = connected_components(A, directed=False)
    return lab == lab[0]


# ---------------------------------------------------------------------------------------------------------------------
# one normal system  B_f^T B_f x = B_f^T c  over the free unknowns
# ---------------------------------------------------------------------------------------------------------------------
@dataclass
class NormalSystem:
    B: Coo                  # least-squares matrix over all unknowns
    target: np.ndarray      # c: min |B x - c| with the gauge's unknowns fixed at x_fix (long double)
    target_mag: np.ndarray  # |c| as evaluated from absolute values
    free: np.ndarray        # boolean mask of the unknowns solved for
    x_fix: np.ndarray       # the fixed unknowns' values (zero off the gauge)
    block: int              # unknowns per pose (d^2 rotations, d translations)
    copies: int             # d: the index l (fastest) of identical decoupled copies (row of R_p, coordinate of t_p)

    def rhs(self):
        """b = B^T (c - B x_fix) on the free unknowns (zero elsewhere), and its absolute evaluation"""
        c = self.target - self.B.mul(self.x_fix)
        cm = self.target_mag + self.B.mul(self.x_fix, absolute=True)
        b, bm = self.B.tmul(c), self.B.tmul(cm, absolute=True)
        b[~self.free], bm[~self.free] = 0, 0
        return b, bm

    def apply(self, x, absolute=False):
        """A x = B^T B x on the free unknowns (x zero off them), or |B|^T |B| |x|"""
        xx = np.where(self.free, ld(x), 0)
        y = self.B.tmul(self.B.mul(xx, absolute), absolute)
        y[~self.free] = 0
        return y

    def diag(self):
        """diag(B^T B): the Jacobi scaling D of the GPU solver"""
        D = np.zeros(self.B.shape[1])
        np.add.at(D, self.B.cols, self.B.vals ** 2)
        return D

    def reduced(self):
        Bc = self.B.csc()[:, np.flatnonzero(self.free)]
        return (Bc.T @ Bc).tocsc()

    def solve(self, max_steps=30):
        """x over all unknowns (x_fix on the gauge, zero outside the component of pose 0), long double.  Refined until a
        correction no longer halves; the last relative correction is kept in `refined_to`."""
        idx = np.flatnonzero(self.free)
        x = ld(self.x_fix).copy()
        self.refined_to = 0.0
        if len(idx) == 0:
            return x
        lu = spla.splu(self.reduced())
        b, _ = self.rhs()
        x[idx] = ld(lu.solve(np.asarray(b[idx], dtype=np.float64)))
        prev = np.inf
        for _ in range(max_steps):
            res = b - self.apply(x)
            dx = ld(lu.solve(np.asarray(res[idx], dtype=np.float64)))
            x[idx] += dx
            step = float(np.max(np.abs(dx)) / max(np.max(np.abs(x[idx])), np.finfo(float).tiny))
            if step == 0.0 or step > 0.5 * prev:
                break
            prev = step
        self.refined_to = step
        return x

    def scaled_extremes(self, want_max=True):
        """(lambda_min, lambda_max) of D^-1/2 A D^-1/2 on the free unknowns (lambda_max None unless want_max).  The
        unknowns of one row l of the rotations (one coordinate l of the translations) form a block that does not couple
        to the others and repeats for every l, so one block is enough."""
        free = self.free & ((np.arange(len(self.free)) % self.copies) == 0)
        idx = np.flatnonzero(free)
        Bc = self.B.csc()[:, idx]
        A = (Bc.T @ Bc).tocsc()
        s = 1.0 / np.sqrt(A.diagonal())
        As = (sp.diags(s) @ A @ sp.diags(s)).tocsc()
        if len(idx) <= DENSE_EIG_MAX:
            ev = np.linalg.eigvalsh(As.toarray())
            return float(ev[0]), float(ev[-1]) if want_max else None
        lmin = float(spla.eigsh(As, k=1, sigma=0.0, which="LM", return_eigenvectors=False, tol=1e-10)[0])
        lmax = float(spla.eigsh(As, k=1, which="LA", return_eigenvectors=False, tol=1e-8)[0]) if want_max else None
        return lmin, lmax


def rotation_system(edges, n) -> NormalSystem:
    """The reference's rotation problem: min |B3 x| with R_0 = I, over the poses joined to pose 0 by kappa > 0."""
    d = edges.d
    d2 = d * d
    comp = component_of_zero(n, edges.p1, edges.p2, edges.kappa)
    free = np.repeat(comp, d2)
    free[:d2] = False
    x_fix = np.zeros(d2 * n)
    x_fix[:d2] = np.eye(d).reshape(-1, order="F")
    return NormalSystem(b3_matrix(edges, n), np.zeros(d2 * len(edges), dtype=LD), np.zeros(d2 * len(edges), dtype=LD),
                        free, x_fix, d2, d)


def translation_system(edges, n, R) -> NormalSystem:
    """The reference's translation problem for the rotations R (n, d, d): min |B1 t - sqrt(tau) R_i t_ij| with t_0 = 0, over
    the poses joined to pose 0 by tau > 0 (free=all: every pose but 0, as the GPU solves it)."""
    d = edges.d
    comp = component_of_zero(n, edges.p1, edges.p2, edges.tau)
    free = np.repeat(comp, d)
    free[:d] = False
    c, cm = b2_target(edges, R)
    return NormalSystem(b1_matrix(edges, n), c, cm, free, np.zeros(d * n), d, d)


def with_free(sys_: NormalSystem, free) -> NormalSystem:
    return NormalSystem(sys_.B, sys_.target, sys_.target_mag, np.asarray(free, dtype=bool), sys_.x_fix, sys_.block,
                        sys_.copies)


def all_but_zero(sys_: NormalSystem) -> NormalSystem:
    """The same problem over every unknown except the gauge's: the (singular when disconnected) system the GPU solves."""
    free = np.ones(len(sys_.free), dtype=bool)
    free[:sys_.block] = False
    return with_free(sys_, free)


# ---------------------------------------------------------------------------------------------------------------------
# the answer
# ---------------------------------------------------------------------------------------------------------------------
def project_to_rotation(M):
    """ref projectToRotationGroup (src/DPGO_utils.cpp:463-477): U V^T, the column of U of the smallest singular value
    negated when det(U V^T) < 0."""
    Um, _, Vt = np.linalg.svd(np.asarray(M, dtype=np.float64))
    if np.linalg.det(Um) * np.linalg.det(Vt) < 0:
        Um = Um.copy()
        Um[:, -1] = -Um[:, -1]
    return Um @ Vt


def unvec_rotations(x, d):
    """(n, d, d) from vec(R_p) column-major"""
    n = len(x) // (d * d)
    return np.transpose(np.asarray(x).reshape(n, d, d), (0, 2, 1))


@dataclass
class Reference:
    M: np.ndarray           # (n, d, d) unprojected rotations, long double (zero outside the component of pose 0)
    R: np.ndarray           # (n, d, d) projected (I outside the component of pose 0)
    t: np.ndarray           # (n, d) long double (zero outside the component of pose 0)
    rot: NormalSystem
    tra: NormalSystem

    def T(self):
        n, d = self.R.shape[0], self.R.shape[1]
        T = np.zeros((d, (d + 1) * n))
        for p in range(n):
            T[:, p * (d + 1):p * (d + 1) + d] = self.R[p]
            T[:, p * (d + 1) + d] = np.asarray(self.t[p], dtype=np.float64)
        return T


def chordal_reference(edges, n) -> Reference:
    d = edges.d
    rot = rotation_system(edges, n)
    M = unvec_rotations(rot.solve(), d)
    R = np.array([project_to_rotation(M[p]) if rot.free[p * d * d] or p == 0 else np.eye(d) for p in range(n)])
    tra = translation_system(edges, n, R)
    t = tra.solve().reshape(n, d)
    return Reference(M, R, t, rot, tra)


def split_T(T, d):
    """(R (n, d, d), t (n, d)) of a d x (d+1) n trajectory"""
    n = T.shape[1] // (d + 1)
    Tt = np.asarray(T).reshape(d, n, d + 1)
    return np.transpose(Tt[:, :, :d], (1, 0, 2)), Tt[:, :, d].T.copy()


# ---------------------------------------------------------------------------------------------------------------------
# bounds
# ---------------------------------------------------------------------------------------------------------------------
def row_blocks(edges, n):
    """distinct blocks of each block row of the normal matrices (the diagonal block and one per neighbour)"""
    key = np.unique(np.concatenate([np.asarray(edges.p1) * n + edges.p2, np.asarray(edges.p2) * n + edges.p1,
                                    np.arange(n) * (n + 1)]))
    return np.bincount(key // n, minlength=n)


def gap_constant(edges, n):
    """c of the residual bound: twice the forward-error constant (K + 2) of the longest row's product (dot length K =
    3 x blocks, the solver's 3 x 3 container blocks), once for the product of the returned iterate and once for the drift
    of the recursive residual from the true one."""
    return 2.0 * (3.0 * float(row_blocks(edges, n).max()) + 2.0)


def _dnorm(v, D, free):
    v = np.asarray(v, dtype=LD)[free]
    return float(np.sqrt(np.sum(v * v / ld(D[free]))))


def residual_bound(sys_: NormalSystem, x, tol, c):
    """tol ||D^-1/2 b|| + c u (||D^-1/2 |A| |x| || + ||D^-1/2 |b| ||) over the free unknowns with D > 0"""
    D = sys_.diag()
    free = sys_.free & (D > 0)
    b, bm = sys_.rhs()
    Ax = sys_.apply(x, absolute=True)
    return tol * _dnorm(b, D, free) + c * U * (_dnorm(Ax, D, free) + _dnorm(bm, D, free))


def residual_norm(sys_: NormalSystem, x):
    """||D^-1/2 (b - A x)|| over the free unknowns with D > 0, in long double; and whether every free unknown with D = 0
    (a pose without weighted edges) has a zero residual"""
    D = sys_.diag()
    b, _ = sys_.rhs()
    r = b - sys_.apply(x)
    return _dnorm(r, D, sys_.free & (D > 0)), bool(np.all(r[sys_.free & (D == 0)] == 0))


def dweighted_error(sys_: NormalSystem, x, x_ref):
    """||D^1/2 (x - x_ref)|| over the free unknowns"""
    D = sys_.diag()
    e = (ld(x) - ld(x_ref))[sys_.free]
    return float(np.sqrt(np.sum(e * e * ld(D[sys_.free]))))


def rotation_tolerances(rot: NormalSystem, M, tol, c):
    """Per pose of the component of pose 0: the bound on |R_gpu - proj(M_p)|_F, where M (n, d, d) is the unprojected
    answer compared against (the reference's, or a ground truth).  The pre-projection error in the D^1/2-norm is at most
    (the GPU's residual bound + M's own residual) / lambda_min; the projection passes it on with 2 / (sigma_{d-1} + sigma_d)
    (sigma_d signed by det M), less twice that error for the change of the singular values.  NaN where that sum is not
    more than four times the error (the projection is not unique enough to bound); pose 0 is exact."""
    n, d = M.shape[0], M.shape[1]
    d2 = d * d
    out = np.full(n, np.nan)
    out[0] = 0.0
    if not rot.free.any():
        return out
    x = ld(M).transpose(0, 2, 1).reshape(-1)
    lmin, _ = rot.scaled_extremes(want_max=False)
    err = (residual_bound(rot, x, tol, c) + residual_norm(rot, x)[0]) / (0.99 * lmin)    # 0.99: the eigensolver's error
    D = rot.diag().reshape(n, d2)
    for p in range(1, n):
        if not rot.free[p * d2]:
            continue
        dp = err / np.sqrt(D[p].min())                              # |M_gpu - M_p|_F
        Mp = np.asarray(M[p], dtype=np.float64)
        s = np.linalg.svd(Mp, compute_uv=False)
        gap = s[-2] + np.sign(np.linalg.det(Mp)) * s[-1]
        if gap > 4 * dp:
            out[p] = 2.0 * (dp + 8 * d * U * s[0]) / (gap - 2 * dp)    # 8 d u sigma_1: the projection's own rounding
    return out


def translation_check(edges, n, T_gpu, R_against, tol, c, t_against=None):
    """The certificate of the GPU's translations, and their distance to the translations t_against (default: the solution
    of the problem with the rotations R_against) on the component of pose 0.  Returns (residual, its bound, D^1/2-norm
    error, its bound):  the error is at most (the certificate's bound + |D^-1/2 (b(R_against) - b(R_gpu))| + t_against's
    own residual) / lambda_min."""
    d = edges.d
    Rg, tg = split_T(T_gpu, d)
    x = ld(tg).reshape(-1)
    sys_g = all_but_zero(translation_system(edges, n, Rg))
    res, zero_ok = residual_norm(sys_g, x)
    assert zero_ok, "a pose without weighted edges has a nonzero translation residual"
    bound = residual_bound(sys_g, x, tol, c)
    sys_a = translation_system(edges, n, R_against)
    if not sys_a.free.any():
        return res, bound, 0.0, 0.0
    ta = sys_a.solve() if t_against is None else ld(t_against).reshape(-1)
    D = sys_a.diag()
    live = sys_a.free & (D > 0)
    gap = _dnorm(sys_a.rhs()[0] - with_free(sys_g, sys_a.free).rhs()[0], D, live)
    lmin, _ = sys_a.scaled_extremes(want_max=False)
    err = dweighted_error(sys_a, np.where(sys_a.free, x, 0), ta)
    return res, bound, err, (bound + gap + residual_norm(sys_a, ta)[0]) / (0.99 * lmin)

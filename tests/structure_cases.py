"""Pose graphs whose shape reaches the kernels' host-chosen branches, and componentwise comparators against a
high-precision reference.  Helper module of test_structure_cases.py (CPU) and test_gpu_structures.py (GPU), whose graphs
the chordal-initialisation tests (test_chordal_cpu.py, test_gpu_chordal.py) reuse; no fixtures.

The shipped datasets have small, even degrees and no empty rows, so several branches of the library are never taken on
them.  Each case below names the branch it is built for (`Case.target`); test_structure_cases.py checks from host facts
alone that the case really reaches it.

The comparators take the reference in long double from the same doubles the library received, and bound each element
by the standard forward-error bound of its formula: the formula evaluated once more on absolute values, times the dot
lengths, times u.  Such a bound holds for any summation order, so it does not depend on how a kernel reduces.
"""
from __future__ import annotations

import os
import re
from dataclasses import dataclass
from typing import Optional

import numpy as np
import scipy.sparse as sp

from dpo_b200 import posegraph as pg

# mirrored from dpgo_kernels.cuh / nd_precond.h
SPMV_GROUP_BLOCKS = 192      # blocks per row group of the TMA-fed Q.X product; a longer row sends it to the gather kernel
SP_CACHE_INTS = 2048         # a CTA's block-CSR slice (rows + 1 + blocks) beyond this is read from global memory
DENSE_MAX_N = 12000          # the dense exact preconditioner (one macro level) is exercised up to this N ((d+1) n)
U = 2.0 ** -53               # unit roundoff of float64


def _max_rank():
    """DPGO_MAX_RANK of the C header: every d <= r <= DPGO_MAX_RANK is compiled"""
    hdr = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "dpgo_b200.h")
    with open(hdr) as fh:
        return int(re.search(r"^#define DPGO_MAX_RANK (\d+)", fh.read(), re.M).group(1))


MAX_RANK = _max_rank()
RANKS = {d: tuple(range(d, MAX_RANK + 1)) for d in (3, 2)}   # every compiled relaxation rank per d: d <= r <= DPGO_MAX_RANK


def nd_ycap_tiles(r, dh):
    """shared-memory tile capacity of one nested-dissection step at rank r (larger leaves: column chunks)"""
    return 600 if r * dh <= 20 else 12000 // (r * dh)


def nd_slot_cap(r):
    """partial-sum slots of one nested-dissection step at rank r"""
    return 240 if r <= 5 else 1200 // r


@dataclass
class Case:
    name: str
    d: int
    n: int
    edges: pg.EdgeSet
    target: str
    static_pose: Optional[np.ndarray] = None          # prior blocks at (pose, pose)
    static_blocks: Optional[np.ndarray] = None

    @property
    def dh(self):
        return self.d + 1

    @property
    def N(self):
        return self.dh * self.n

    def triplets(self):
        """(brow, bcol, blocks) with duplicates not merged: the edges' four blocks each, then the prior blocks."""
        brow, bcol, blocks = pg.connection_laplacian_blocks(self.edges)
        if self.static_pose is not None and len(self.static_pose):
            sp_ = np.asarray(self.static_pose, dtype=np.int32)
            brow = np.concatenate([brow, sp_])
            bcol = np.concatenate([bcol, sp_])
            blocks = np.concatenate([blocks, np.asarray(self.static_blocks, dtype=np.float64)])
        return brow.astype(np.int32), bcol.astype(np.int32), blocks

    def Q(self) -> sp.csr_matrix:
        """Q in float64 with explicit zeros kept, so that its block pattern is that of the triplets."""
        brow, bcol, blocks = self.triplets()
        dh = self.dh
        k, c = np.meshgrid(np.arange(dh), np.arange(dh), indexing="ij")
        rows = (brow[:, None, None].astype(np.int64) * dh + k[None]).ravel()
        cols = (bcol[:, None, None].astype(np.int64) * dh + c[None]).ravel()
        Q = sp.coo_matrix((blocks.ravel(), (rows, cols)), shape=(self.N, self.N)).tocsr()
        Q.sum_duplicates()
        return Q

    def row_blocks(self) -> np.ndarray:
        """Number of distinct blocks in each block row of Q."""
        brow, bcol, _ = self.triplets()
        key = np.unique(brow.astype(np.int64) * self.n + bcol)
        return np.bincount(key // self.n, minlength=self.n)


# ---------------------------------------------------------------------------------------------------------------------
# graph construction
# ---------------------------------------------------------------------------------------------------------------------
def random_rotations(rng, m, d):
    if d == 2:
        th = rng.uniform(-np.pi, np.pi, m)
        return np.stack([np.stack([np.cos(th), -np.sin(th)], -1), np.stack([np.sin(th), np.cos(th)], -1)], -2)
    Qm, Rm = np.linalg.qr(rng.standard_normal((m, 3, 3)))
    Qm = Qm * np.sign(np.diagonal(Rm, axis1=1, axis2=2))[:, None, :]
    Qm[np.linalg.det(Qm) < 0, :, 0] *= -1.0
    return Qm


def edge_set(rng, d, pairs):
    pairs = np.asarray(pairs, dtype=np.int64).reshape(-1, 2)
    m = len(pairs)
    z = np.zeros(m, dtype=np.int64)
    return pg.EdgeSet(d, z, z, pairs[:, 0], pairs[:, 1], random_rotations(rng, m, d), rng.standard_normal((m, d)),
                      rng.uniform(1.0, 100.0, m), rng.uniform(0.5, 10.0, m))


def noise_free_graph(d, pairs, n, seed=0, kappa=None, tau=None):
    """Random ground-truth poses and the exact relative measurements of `pairs` between them; weights as edge_set draws
    them unless given.  Returns (n, edges, ground-truth T of shape (d, (d+1) n))."""
    rng = np.random.default_rng([seed, d, n])
    Rp = random_rotations(rng, n, d)
    tp = rng.uniform(-10.0, 10.0, (n, d))
    e = edge_set(rng, d, pairs)
    i, j = e.p1, e.p2
    e.R[:] = np.einsum("mba,mbc->mac", Rp[i], Rp[j])                  # R_i^T R_j
    e.t[:] = np.einsum("mba,mb->ma", Rp[i], tp[j] - tp[i])            # R_i^T (t_j - t_i)
    if kappa is not None:
        e.kappa[:] = kappa
    if tau is not None:
        e.tau[:] = tau
    T = np.concatenate([Rp, tp[:, :, None]], axis=2)                  # (n, d, d+1)
    return n, e, np.transpose(T, (1, 0, 2)).reshape(d, (d + 1) * n)


def in_gauge_of_pose_zero(T, d):
    """T expressed in the frame of its pose 0 (R_0 = I, t_0 = 0)."""
    n = T.shape[1] // (d + 1)
    Tt = np.asarray(T).reshape(d, n, d + 1)
    R0, t0 = Tt[:, 0, :d], Tt[:, 0, d]
    out = np.einsum("ba,bnc->anc", R0, Tt)
    out[:, :, d] = np.einsum("ba,bn->an", R0, Tt[:, :, d] - t0[:, None])
    return out.reshape(d, (d + 1) * n)


def chain(poses):
    poses = list(poses)
    return [(poses[i], poses[i + 1]) for i in range(len(poses) - 1)]


def star_with_leaf_chain(leaves, leaf_chain=True):
    pairs = [(0, i) for i in range(1, leaves + 1)]
    if leaf_chain:
        pairs += chain(range(1, leaves + 1))
    return pairs


def _tail_isolated():
    interior = {60, 130, 131}
    active = [i for i in range(205) if i not in interior]       # 202 poses: 3 * 202 - 2 = 604 blocks, a multiple of 4
    return 205 + 420, chain(active)


def _clique(n):
    """every pair once: no separator, so the nested dissection keeps one leaf of n poses"""
    i, j = np.triu_indices(n, 1)
    return np.stack([i, j], 1)


def _multi_edges(rng):
    base = chain(range(40))
    dup = [(5, 6), (5, 6), (12, 13)]                     # duplicated edges
    rev = [(21, 20), (30, 29)]                           # p1 > p2
    both = [(8, 9), (9, 8), (33, 34), (34, 33)]          # both directions between the same pair
    rnd = [(40 + int(a), 40 + int(b)) for a, b in rng.integers(0, 300, size=(700, 2)) if a != b]
    return 340, base + dup + rev + both + rnd


CASE_NAMES = ("single", "single_prior", "pair", "triple", "hub191", "hub192", "hub2100", "tail_isolated", "components",
              "clique700", "multi_edges", "long_chain")
LARGE = ("hub2100", "long_chain")             # run with r in large_ranks(d) only, as clique700


def large_ranks(d):
    """the ranks the largest cases run at: d, the largest rank of the fixed capacities (5) and DPGO_MAX_RANK"""
    return (d, 5, MAX_RANK)


def make_case(name: str, d: int, seed: int = 0) -> Case:
    rng = np.random.default_rng([seed, d, CASE_NAMES.index(name)])
    static = None
    if name == "single":
        n, pairs, target = 1, [], "n = 1, nb = 0: no row groups, most CTAs of the full grid own nothing"
    elif name == "single_prior":
        n, pairs, target = 1, [], "n = 1 with one prior block: one row group of one block"
        M = rng.standard_normal((d + 1, d + 1))
        static = (np.array([0]), (M @ M.T + np.eye(d + 1))[None])
    elif name == "pair":
        n, pairs, target = 2, [(0, 1)], "n = 2"
    elif name == "triple":
        n, pairs, target = 3, chain(range(3)), "n = 3 path"
    elif name == "hub191":
        n, pairs, target = 192, star_with_leaf_chain(191), "hub row of exactly 192 blocks: one full TMA stage"
    elif name == "hub192":
        n, pairs, target = 193, star_with_leaf_chain(192), "hub row of 193 blocks: stand-alone Q.X on the gather kernel"
    elif name == "hub2100":
        n, pairs, target = 2101, star_with_leaf_chain(2100, leaf_chain=False), \
            "hub row of 2101 blocks: its CTA reads the block-CSR from global memory; ND: star, 2100 singleton leaves"
    elif name == "tail_isolated":
        (n, pairs), target = _tail_isolated(), "interior and trailing empty rows, nb % 4 == 0: 0-byte index windows"
    elif name == "components":
        n = 67
        pairs = chain(range(30)) + chain(range(30, 60)) + [(i, j) for i in range(61, 67) for j in range(i + 1, 67)]
        target = "two chains, an isolated pose and a clique, no edges between them"
    elif name == "clique700":
        n = 700 if d == 3 else 701
        pairs = _clique(n)
        target = "ND leaf > nd_ycap_tiles at every rank; n even (N = 2800) and odd (N = 2103: the last panel half used)"
    elif name == "multi_edges":
        (n, pairs), target = _multi_edges(rng), "duplicated and reversed edges, both directions, random sparse part"
    elif name == "long_chain":
        n, pairs, target = 5000, chain(range(5000)), "5000-pose path: deep dissection"
    else:
        raise KeyError(name)
    edges = edge_set(rng, d, pairs) if len(pairs) else pg.EdgeSet.empty(d)
    c = Case(name, d, n, edges, target)
    if static is not None:
        c.static_pose, c.static_blocks = static
    return c


# ---------------------------------------------------------------------------------------------------------------------
# host facts: which branch a case reaches
# ---------------------------------------------------------------------------------------------------------------------
def tma_groups(row_blocks, bt=SPMV_GROUP_BLOCKS):
    """Row groups of the TMA-fed product as the library cuts them (build_from_triplets in dpgo_capi.cu): consecutive rows,
    <= bt rows and <= bt blocks each.  [(row0, row1, block0, block1)], or None when a row exceeds bt blocks or Q has
    no block (the gather kernel runs then)."""
    rowptr = np.concatenate([[0], np.cumsum(row_blocks)])
    n = len(row_blocks)
    out, rr = [], 0
    while rr < n:
        start, blocks = rr, 0
        while rr < n and rr - start < bt and blocks + row_blocks[rr] <= bt:
            blocks += row_blocks[rr]
            rr += 1
        if rr == start:
            return None
        out.append((start, rr, int(rowptr[start]), int(rowptr[rr])))
    return out if rowptr[-1] > 0 else None


def zero_byte_index_groups(groups):
    """Groups without blocks whose first block index is a multiple of 4: their index window is empty."""
    return [g for g in (groups or []) if g[2] == g[3] and g[2] % 4 == 0]


# ---------------------------------------------------------------------------------------------------------------------
# references and componentwise bounds
# ---------------------------------------------------------------------------------------------------------------------
LD = np.longdouble


def ld(a):
    return np.asarray(a, dtype=LD)


def tiles(X, d):
    r, N = X.shape
    return X.reshape(r, N // (d + 1), d + 1)


def pose_K(case_or_rowblocks, d):
    """K_j = (d+1) * blocks(row j): the length of every dot product that makes column block j of X Q."""
    rb = case_or_rowblocks.row_blocks() if isinstance(case_or_rowblocks, Case) else np.asarray(case_or_rowblocks)
    return (d + 1) * rb


def per_elem(kpose, r, d):
    """per-pose numbers broadcast to the (r, (d+1) n) layout"""
    return np.broadcast_to(np.repeat(np.asarray(kpose, dtype=np.float64), d + 1)[None, :], (r, (d + 1) * len(kpose)))


def product_ref(Q, X, G=None):
    """X Q (+ G) in long double from the same doubles, and the bound's magnitude |X| |Q| (+ |G|)"""
    Ql = sp.csr_matrix(Q).astype(LD)
    ref = (Ql @ ld(X).T).T
    mag = (abs(Ql) @ abs(ld(X)).T).T
    if G is not None:
        ref = ref + ld(G)
        mag = mag + abs(ld(G))
    return ref, mag


def check_product(got, Q, X, K, G=None, what="X Q"):
    """|got - ref| <= (K_j + 2) u (|X| |Q| + |G|) per element, for any summation order (fma or DMMA included)."""
    r, N = X.shape
    ref, mag = product_ref(Q, X, G)
    bound = (per_elem(K, r, N // len(K) - 1) + 2.0) * U * mag
    err = abs(ld(got) - ref)
    bad = err > bound
    assert not bad.any(), f"{what}: {int(bad.sum())} elements out of bound, worst at {np.unravel_index(np.argmax(err - bound), err.shape)}: " \
                          f"err {float(err.max()):.3e}, bound there {float(bound.ravel()[np.argmax(err - bound)]):.3e}"


def _proj(Y, Z, d, plus=False):
    """tangent projection Z_Y - Y sym(Y^T Z_Y) on tiles; with plus=True the absolute-value evaluation (inputs already
    absolute): Z_Y + Y (Y^T Z + Z^T Y) / 2"""
    Yt, Zt = tiles(Y, d), tiles(Z, d)
    Yr, Zr = Yt[:, :, :d], Zt[:, :, :d]
    S = np.einsum("ani,anj->nij", Yr, Zr)
    S = (S + np.transpose(S, (0, 2, 1))) / 2
    out = Zt.copy()
    corr = np.einsum("ani,nij->anj", Yr, S)
    out[:, :, :d] = Zr + corr if plus else Zr - corr
    return out.reshape(Z.shape)


def projection_ref(X, Z, d):
    return _proj(ld(X), ld(Z), d), _proj(abs(ld(X)), abs(ld(Z)), d, plus=True)


def check_elementwise(got, ref, mag, c, what):
    """|got - ref| <= c u mag per element (c: scalar or per-element array)"""
    bound = np.asarray(c, dtype=np.float64) * U * mag
    err = abs(ld(got) - ref)
    bad = err > bound
    assert not bad.any(), f"{what}: {int(bad.sum())} elements out of bound, worst err {float(err.max()):.3e}, " \
                          f"at {np.unravel_index(np.argmax(err - bound), err.shape)}"


def stage_c(K, r, d):
    """constant of a composed formula: the product's K_j + 2 plus the dot lengths of a projection (r, d), twice over
    (first-order bound of a composition of two such stages)"""
    return 2.0 * (per_elem(K, r, d) + 2 * r + 2 * d + 6)


def rgrad_ref(Q, G, X, d):
    EG, EGm = product_ref(Q, X, G)
    return _proj(ld(X), EG, d), _proj(abs(ld(X)), EGm, d, plus=True), EG, EGm


def rhess_ref(Q, G, X, V, d):
    """P_X(V Q - V_Y sym(Y^T EG_Y)) and its absolute-value evaluation"""
    _, _, EG, EGm = rgrad_ref(Q, G, X, d)
    HV, HVm = product_ref(Q, V)
    out = []
    for Xs, Vs, Es, Hs, plus in ((ld(X), ld(V), EG, HV, False), (abs(ld(X)), abs(ld(V)), EGm, HVm, True)):
        Yt, Et, Vt = tiles(Xs, d), tiles(Es, d), tiles(Vs, d)
        S = np.einsum("ani,anj->nij", Yt[:, :, :d], Et[:, :, :d])
        S = (S + np.transpose(S, (0, 2, 1))) / 2
        Ht = tiles(Hs, d).copy()
        corr = np.einsum("ani,nij->anj", Vt[:, :, :d], S)
        Ht[:, :, :d] = Ht[:, :, :d] + corr if plus else Ht[:, :, :d] - corr
        out.append(_proj(Xs, Ht.reshape(X.shape), d, plus=plus))
    return out[0], out[1]


def f_ref(Q, G, X):
    XQ, XQm = product_ref(Q, X)
    Xl = ld(X)
    val = 0.5 * np.sum(XQ * Xl) + np.sum(Xl * ld(G))
    mag = 0.5 * np.sum(XQm * abs(Xl)) + np.sum(abs(Xl) * abs(ld(G)))
    return val, mag


def check_scalar(got, ref, mag, K, count, what):
    """|got - ref| <= (max K + count + 2) u mag: a sum of `count` terms in any order after the products"""
    bound = (float(np.max(K, initial=0)) + count + 2.0) * U * float(mag)
    assert abs(LD(got) - ref) <= bound, f"{what}: {got!r} vs {float(ref)!r}, err {float(abs(LD(got) - ref)):.3e} > {bound:.3e}"


def jacobi_ref(Q, X, V, d):
    """P_X(V D^-1) with D = blockdiag(Q_jj + 0.1 I) inverted in long double, its magnitude and the blocks' condition numbers"""
    dh = d + 1
    n = Q.shape[0] // dh
    Qb = sp.csr_matrix(Q).tobsr(blocksize=(dh, dh))
    Dinv = np.zeros((n, dh, dh), dtype=LD)
    cond = np.ones(n)
    for i in range(n):
        blk = np.zeros((dh, dh))
        for k in range(Qb.indptr[i], Qb.indptr[i + 1]):
            if Qb.indices[k] == i:
                blk = Qb.data[k].copy()
        A = blk + 0.1 * np.eye(dh)
        cond[i] = np.linalg.cond(A)
        Dinv[i] = _ld_inverse(ld(A))
    Vt = tiles(ld(V), d)
    Z = np.einsum("ank,nkc->anc", Vt, Dinv).reshape(V.shape)
    Zm = np.einsum("ank,nkc->anc", abs(Vt), abs(Dinv)).reshape(V.shape)
    P, Pm = _proj(ld(X), Z, d), _proj(abs(ld(X)), Zm, d, plus=True)
    return P, Pm, cond


def _ld_inverse(A):
    """Gauss-Jordan with partial pivoting in long double (numpy's inverse has no long-double kernel)"""
    m = A.shape[0]
    M = np.concatenate([A.copy(), np.eye(m, dtype=LD)], axis=1)
    for c in range(m):
        p = c + int(np.argmax(abs(M[c:, c])))
        M[[c, p]] = M[[p, c]]
        M[c] /= M[c, c]
        for rr in range(m):
            if rr != c:
                M[rr] -= M[rr, c] * M[c]
    return M[:, m:]


def exact_ref(Q, X, V, d, shift=0.1):
    """P_X(A^-1 V) with A = Q + 0.1 I: sparse LU plus one refinement step with the residual in long double; and
    kappa(A) <= (lambda_max(Q) + 0.1) / 0.1 (Q is positive semi-definite)"""
    import scipy.sparse.linalg as spla
    N = Q.shape[0]
    A = (sp.csr_matrix(Q) + shift * sp.identity(N, format="csr")).tocsc()
    lu = spla.splu(A)
    Z = lu.solve(np.ascontiguousarray(V.T))
    Al = A.astype(LD)
    res = ld(V.T) - Al @ ld(Z)
    Zl = ld(Z) + ld(lu.solve(np.asarray(res, dtype=np.float64)))
    if N > 64:
        lmax = float(spla.eigsh(sp.csr_matrix(Q), k=1, which="LA", return_eigenvectors=False, tol=1e-3)[0]) * 1.01
    else:
        lmax = float(np.linalg.eigvalsh(sp.csr_matrix(Q).toarray()).max()) if N else 0.0
    kappa = (max(lmax, 0.0) + shift) / shift
    return _proj(ld(X), Zl.T, d), kappa


def check_exact(got, ref, kappa, d, c, what):
    """per tile: max tile error over max tile norm <= c u kappa; globally: relative Frobenius error <= c u kappa"""
    e = np.asarray(ld(got) - ref, dtype=np.float64)
    rf = np.asarray(ref, dtype=np.float64)
    te = np.sqrt((tiles(e, d) ** 2).sum(axis=(0, 2)))
    tn = np.sqrt((tiles(rf, d) ** 2).sum(axis=(0, 2)))
    tol = c * U * kappa
    assert te.max() <= tol * max(tn.max(), 1e-300), f"{what}: worst tile {int(te.argmax())} err {te.max():.3e} " \
                                                     f"vs {tol:.2e} * {tn.max():.3e}"
    assert np.linalg.norm(e) <= tol * np.linalg.norm(rf), f"{what}: global {np.linalg.norm(e) / np.linalg.norm(rf):.3e} > {tol:.2e}"

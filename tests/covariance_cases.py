"""Pose graphs whose shape takes the pose-covariance path (dpgo_pose_covariances) where the datasets never go, an
extended-precision reference of the covariance, and the element-wise bound a result must meet.  Helper module of
test_covariance_cases_cpu.py (host emulation, no GPU) and test_gpu_covariance_cases.py (device); no fixtures.

Each case names the regime it is built for (`CovCase.target`); the CPU test checks from the planner's host facts
(info16) that the case really reaches it.

Reference.  H is formed in long double from the same doubles the library receives, by the model of covariance_oracle
(the Jacobians re-formed in long double, not the fp64 H cast).  Free dimensions up to DENSE_LD_MAX are inverted densely
in long double (NumPy has no long-double LAPACK, so the Gauss-Jordan is a Python loop and this stays small); larger ones
by fp64 splu column solves with two refinement steps whose residuals come from the long-double H, at SAMPLE poses and
every requested pair.

Bound.  With H_f the anchored information, D = diag(H_f), H^ = D^-1/2 H_f D^-1/2 and k^ = lmax(H^) / lmin(H^), element
(a, c) of every block must satisfy
    |Sigma[a, c] - Sigma_ref[a, c]| <= C u k^ ||H^^-1||_2 / sqrt(h_aa h_cc),    u = 2^-53,
which follows from conditioning (Sigma = D^-1/2 H^^-1 D^-1/2, so |Sigma[a, c]| <= ||H^^-1|| / sqrt(h_aa h_cc)) and holds for
any factorisation that is backward stable on the scaled matrix.  One constant C for every case.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, Optional

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

import covariance_oracle as co
import structure_cases as sc
from dpo_b200 import posegraph as pg

LD = np.longdouble
U = 2.0 ** -53                 # unit roundoff of float64
C_BOUND = 64.0                 # the bound's constant, for every case
DENSE_LD_MAX = 400             # free dimensions up to this are inverted densely in long double
DENSE_EIG_MAX = 3000           # scaled information up to this dimension gets dense eigenvalues
SAMPLE = 64                    # poses sampled (with every requested pair) where the reference is a column solve
MAX_GRID_YZ = 65535            # dpgo_kernels.cuh: nodes of one stage per launch


@dataclass
class CovCase:
    name: str
    d: int
    n: int
    edges: pg.EdgeSet
    T: np.ndarray                                   # d x (d+1) n
    anchor: int
    pairs: np.ndarray                               # (k, 2) int32
    target: str
    closed: Dict[int, np.ndarray] = field(default_factory=dict)    # pose -> its block in closed form
    watch: tuple = ()                               # poses every reference sample includes

    @property
    def b(self):
        return co.tangent_dim(self.d)

    @property
    def id(self):
        return f"{self.name}-{self.d}d"


# ---------------------------------------------------------------------------------------------------------------------
# graphs
# ---------------------------------------------------------------------------------------------------------------------
def _rot(d, w):
    """rotations exp([w]x) of the rows of w ((k, 1) in 2D, (k, 3) in 3D), vectorised"""
    if d == 2:
        c, s = np.cos(w[:, 0]), np.sin(w[:, 0])
        return np.stack([np.stack([c, -s], -1), np.stack([s, c], -1)], -2)
    th = np.linalg.norm(w, axis=1)
    K = np.einsum("mk,kab->mab", w, co.generators(3))
    a = np.where(th > 1e-12, np.sin(th) / np.maximum(th, 1e-300), 1.0)
    b = np.where(th > 1e-12, (1 - np.cos(th)) / np.maximum(th, 1e-300) ** 2, 0.5)
    return np.eye(3) + a[:, None, None] * K + b[:, None, None] * (K @ K)


def perturbed(T, d, rng, sigma=0.02):
    """T with every pose moved by a random right perturbation: not a critical point of the measurements"""
    n = T.shape[1] // (d + 1)
    Tp = np.asarray(T).reshape(d, n, d + 1).transpose(1, 0, 2).copy()         # (n, d, d+1)
    nw = 3 if d == 3 else 1
    x = sigma * rng.standard_normal((n, nw + d))
    R = Tp[:, :, :d].copy()
    Tp[:, :, :d] = R @ _rot(d, x[:, :nw])
    Tp[:, :, d] += np.einsum("nab,nb->na", R, x[:, nw:])
    return np.ascontiguousarray(Tp.transpose(1, 0, 2).reshape(d, (d + 1) * n))


def consistent(d, pairs, n, seed, perturb=True, kappa=None, tau=None):
    """edges measured exactly between random ground-truth poses; T the ground truth, perturbed unless told otherwise"""
    n, e, T = sc.noise_free_graph(d, pairs, n, seed=seed, kappa=kappa, tau=tau)
    if perturb:
        T = perturbed(T, d, np.random.default_rng([seed, d, 1]))
    return e, T


def lattice(k):
    """k x k grid, poses row by row, right and down neighbours"""
    idx = np.arange(k * k).reshape(k, k)
    return [(int(a), int(b)) for a, b in zip(idx[:, :-1].ravel(), idx[:, 1:].ravel())] + \
           [(int(a), int(b)) for a, b in zip(idx[:-1, :].ravel(), idx[1:, :].ravel())]


def _leaf_closed_form(edges, b, d):
    """A pose that ends (p2) exactly one edge and touches no other has the block diag(1 / (2 kappa w) .., 1 / (tau w) ..) when
    the other end is the anchor: d r_rot / d w_j = R_j G_k and d r_tra / d v_j = R_j e_k do not depend on the measurement
    or couple w_j to v_j, at any trajectory."""
    nw = 3 if d == 3 else 1
    return {int(edges.p2[e]): np.diag([1 / (2 * edges.kappa[e] * edges.weight[e])] * nw +
                                      [1 / (edges.tau[e] * edges.weight[e])] * d) for e in range(len(edges))}


def _connect(n, pairs):
    """`pairs` plus one edge from pose 0's component to the smallest pose of every other component"""
    pr = np.asarray(pairs, dtype=np.int64)
    A = sp.coo_matrix((np.ones(len(pr)), (pr[:, 0], pr[:, 1])), shape=(n, n))
    _, lab = sp.csgraph.connected_components(A, directed=False)
    extra = [(0, int(np.flatnonzero(lab == c)[0])) for c in np.unique(lab) if c != lab[0]]
    return [tuple(map(int, p)) for p in pr] + extra


def _graded(d, seed):
    """the 30 x 30 lattice with kappa and tau graded over 1e-6 .. 1e6 along x and weights over 1e-8 .. 1 along y (each
    edge at its midpoint, with a random factor in [1/2, 2]; kappa and tau together, since a 3D rotation about the lever
    arm is held by kappa alone, so kappa << tau is singular in all but name): the diagonal of H spans
    many orders of magnitude while neighbouring poses differ by little, so the unscaled condition number is enormous and
    the Jacobi-scaled one is not.  Pose 465's four edges end there (p2) with kappa = 1e-6 and weight 1, so its rotation is
    held by that tiny kappa alone (a p2's rotation does not enter the translation residual)."""
    k, p = 30, 465
    pairs = [(a, b_) if b_ == p or a != p else (b_, a) for a, b_ in lattice(k)]
    rng = np.random.default_rng([seed, d, 77])
    m = len(pairs)
    pr = np.asarray(pairs)
    x, y = (pr % k).mean(1) / (k - 1), (pr // k).mean(1) / (k - 1)
    kappa = 10.0 ** (-6 + 12 * x) * 2.0 ** rng.uniform(-1, 1, m)
    tau = 10.0 ** (-6 + 12 * x) * 2.0 ** rng.uniform(-1, 1, m)
    w = 10.0 ** (-8 * y) * 2.0 ** rng.uniform(-1, 0, m)
    mine = pr[:, 1] == p
    kappa[mine], w[mine] = 1e-6, 1.0
    e, T = consistent(d, pairs, k * k, seed, kappa=kappa, tau=tau)
    e.weight = w
    return e, T


def _pairs_2000(rng, n, anchor):
    far = [tuple(map(int, rng.choice(n, 2, replace=False))) for _ in range(300)]
    extra = [(17, 17), (1200, 1200), far[0][::-1], far[1][::-1], far[2], (anchor, 700), (900, anchor), (anchor, anchor)]
    return np.asarray(far + extra, dtype=np.int32)


def make_case(name: str, d: int, seed: int = 0) -> CovCase:
    rng = np.random.default_rng([seed, d, sum(map(ord, name))])
    anchor, pairs, closed = 0, [], {}
    if name == "single":
        n, e, T = 1, pg.EdgeSet.empty(d), np.concatenate([np.eye(d), np.zeros((d, 1))], 1)
        pairs, target = [(0, 0)], "n = 1: the early return, zeros and OK without a device"
    elif name == "pair":
        n = 2
        e, T = consistent(d, [(0, 1)], n, seed, perturb=False)
        closed = _leaf_closed_form(e, co.tangent_dim(d), d)
        pairs, target = [(1, 1), (0, 1)], "n = 2 at the measurement: Sigma_1 = diag(1 / (2 kappa) .., 1 / tau ..)"
    elif name == "pair_multi":
        n = 2
        e, T = consistent(d, [(0, 1), (0, 1), (1, 0)], n, seed)
        pairs, target = [(1, 1), (1, 0)], "n = 2, 0 -> 1 twice and 1 -> 0 once: contributions summed over duplicated and reversed edges"
    elif name == "triangle":
        n, anchor = 3, 1
        e, T = consistent(d, [(0, 1), (1, 2), (2, 0)], n, seed)
        pairs, target = [(0, 2), (2, 0), (1, 2)], "the smallest graph with a cycle, anchored at pose 1"
    elif name in ("hub2100_anchor_hub", "hub2100_anchor_leaf"):
        n = 2101
        e, T = consistent(d, sc.star_with_leaf_chain(2100, leaf_chain=False), n, seed)
        if name.endswith("hub"):
            closed = _leaf_closed_form(e, co.tangent_dim(d), d)
            target = "anchored at the hub: block-diagonal information, every macro node without boundary, no sweep GEMM"
        else:
            anchor = 1
            target = "anchored at a leaf: every front's boundary is the hub"
    elif name in ("star191_chain_hub", "star191_chain_leaf"):
        n = 192
        e, T = consistent(d, sc.star_with_leaf_chain(191), n, seed)
        anchor = 0 if name.endswith("hub") else 96
        target = "hub with a chain through its leaves: one dense root front in 2D, two levels in 3D"
    elif name.startswith("path5000_a"):
        n, anchor = 5000, int(name[len("path5000_a"):])
        e, T = consistent(d, sc.chain(range(n)), n, seed)
        target = "5000-pose path: deep dissection, badly conditioned"
    elif name in ("clique60", "clique200"):
        n = int(name[6:])
        e, T = consistent(d, sc._clique(n), n, seed)
        target = "every pair an edge: one root front, no boundary"
    elif name == "lattice30x30":
        n = 900
        e, T = consistent(d, lattice(30), n, seed)
        target = "30 x 30 lattice: boundaries past SEL_K = 32 and SEL_T = 64, a multiple of neither"
    elif name == "path2000_pairs":
        n, anchor = 2000, 1000
        e, T = consistent(d, sc.chain(range(n)), n, seed)
        pairs = _pairs_2000(rng, n, anchor)
        target = "300 long-range pairs on a path, plus (i, i), both orders, a duplicate and pairs with the anchor"
    elif name == "graded":
        n, anchor = 900, 29                  # the corner of the largest precisions and weights: the rest hangs off it
        e, T = _graded(d, seed)
        target = "lattice with precisions over 1e-6 .. 1e6 and weights over 1e-8 .. 1: ill-conditioned, not singular"
    elif name == "multi_edges":
        s = sc.make_case("multi_edges", d)
        n = s.n
        pr = _connect(n, np.stack([s.edges.p1, s.edges.p2], 1))
        extra = len(pr) - len(s.edges)
        e = pg.EdgeSet.join([s.edges, sc.edge_set(rng, d, pr[len(s.edges):])]) if extra else s.edges
        T = perturbed(co.random_trajectory(d, n, rng), d, rng)
        target = "duplicated and reversed edges, both directions, random sparse part (measurements unrelated to T)"
    elif name == "path600k":
        n = 600_000
        e, T = consistent(d, sc.chain(range(n)), n, seed)
        target = "600000-pose path: a stage of more than 65535 macro nodes"
    else:
        raise KeyError(name)
    watch = (435, 464, 465, 466, 495) if name == "graded" else ()          # the tiny-kappa pose and its neighbours
    return CovCase(name, d, n, e, T, anchor, np.asarray(pairs, dtype=np.int32).reshape(-1, 2), target, closed, watch)


CASE_NAMES = ("single", "pair", "pair_multi", "triangle", "hub2100_anchor_hub", "hub2100_anchor_leaf", "star191_chain_hub",
              "star191_chain_leaf", "path5000_a0", "path5000_a2500", "path5000_a4999", "clique60", "clique200",
              "lattice30x30", "path2000_pairs", "graded", "multi_edges")
CASES = [(name, d) for name in CASE_NAMES for d in (2, 3)] + [("path600k", 2)]


# ---------------------------------------------------------------------------------------------------------------------
# the library's calls
# ---------------------------------------------------------------------------------------------------------------------
def _args(case: CovCase, edges=None):
    from dpo_b200 import _capi as capi
    e = case.edges if edges is None else edges
    arr = co.edge_arrays(e)
    pr = np.ascontiguousarray(case.pairs, dtype=np.int32)
    return capi, arr, pr, np.asfortranarray(case.T)


def call_device(case: CovCase, edges=None, device=0):
    """dpgo_pose_covariances: (code, cov (n, b, b), pair blocks (k, b, b), info16)"""
    import ctypes as C
    capi, (p1, p2, R, t, kappa, tau, w), pr, Tf = _args(case, edges)
    b = case.b
    cov = np.full((case.n, b, b), np.nan)
    pc = np.full((max(len(pr), 1), b, b), np.nan)
    info = (C.c_int64 * 16)()
    code = capi.load_library().dpgo_pose_covariances(case.n, case.d, len(p1), capi.iptr(p1), capi.iptr(p2), capi.dptr(R), capi.dptr(t),
                                                     capi.dptr(kappa), capi.dptr(tau), capi.dptr(w), capi.dptr(Tf), case.anchor,
                                                     device, len(pr), capi.iptr(pr), capi.dptr(cov), capi.dptr(pc), info)
    return code, cov, pc[:len(pr)], list(info)


def emulate(case: CovCase):
    """dpgo_pose_covariances_debug_emulate with the planner's default options (those of the device call)"""
    import ctypes as C
    capi, (p1, p2, R, t, kappa, tau, w), pr, Tf = _args(case)
    b = case.b
    cov = np.zeros((case.n, b, b))
    pc = np.zeros((max(len(pr), 1), b, b))
    info = (C.c_int64 * 16)()
    capi.check(capi.load_library().dpgo_pose_covariances_debug_emulate(
        case.n, case.d, len(p1), capi.iptr(p1), capi.iptr(p2), capi.dptr(R), capi.dptr(t), capi.dptr(kappa), capi.dptr(tau),
        capi.dptr(w), capi.dptr(Tf), case.anchor, -1, 0, len(pr), capi.iptr(pr), capi.dptr(cov), capi.dptr(pc), info))
    return cov, pc[:len(pr)], list(info)


# ---------------------------------------------------------------------------------------------------------------------
# reference
# ---------------------------------------------------------------------------------------------------------------------
class _LdEdges:
    """an EdgeSet's measurements in long double, for covariance_oracle.jacobians"""

    def __init__(self, e):
        self.d, self.p1, self.p2 = e.d, e.p1, e.p2
        self.R, self.t = e.R.astype(LD), e.t.astype(LD)

    def __len__(self):
        return len(self.p1)


class Reference:
    """Sigma of a case in extended precision, and the conditioning its bound needs."""

    def __init__(self, case: CovCase):
        self.case = case
        d, n, b, e = case.d, case.n, case.b, case.edges
        self.f = co.free_index(n, b, case.anchor)
        nf = len(self.f)
        Ji, Jj = co.jacobians(case.T.astype(LD), _LdEdges(e))
        om = np.concatenate([np.repeat((e.weight.astype(LD) * e.kappa.astype(LD))[:, None], d * d, 1),
                             np.repeat((e.weight.astype(LD) * e.tau.astype(LD))[:, None], d, 1)], axis=1)
        # H_f as b x b blocks over the free poses (the anchor's index -1), summed in long double, sorted by block row
        self.nfp = nfp = n - 1
        fp = np.arange(n) - (np.arange(n) > case.anchor)
        fp[case.anchor] = -1
        keys, vals = [], []
        for A, pa in ((Ji, e.p1), (Jj, e.p2)):
            for B, pc in ((Ji, e.p1), (Jj, e.p2)):
                keep = (fp[pa] >= 0) & (fp[pc] >= 0)
                keys.append(fp[pa][keep] * nfp + fp[pc][keep])
                vals.append(np.einsum("mra,mr,mrc->mac", A[keep], om[keep], B[keep]))
        uk, inv = np.unique(np.concatenate(keys), return_inverse=True)
        self.Hb = np.zeros((len(uk), b, b), dtype=LD)
        np.add.at(self.Hb, inv, np.concatenate(vals))
        self.br, self.bc = uk // max(nfp, 1), uk % max(nfp, 1)
        self.bptr = np.concatenate([[0], np.cumsum(np.bincount(self.br, minlength=nfp))])
        r = (self.br[:, None, None] * b + np.arange(b)[None, :, None] + 0 * np.arange(b)[None, None, :]).ravel()
        c = (self.bc[:, None, None] * b + np.arange(b)[None, None, :] + 0 * np.arange(b)[None, :, None]).ravel()
        self.Hf = sp.csr_matrix((self.Hb.astype(np.float64).ravel(), (r, c)), shape=(nf, nf))
        on = self.br == self.bc
        self.h = np.zeros(nf)
        self.h[(self.br[on][:, None] * b + np.arange(b)).ravel()] = np.diagonal(self.Hb[on], axis1=1, axis2=2).astype(np.float64).ravel()
        self.dense = nf <= DENSE_LD_MAX
        self._S = None
        self._extremes()

    def _extremes(self):
        """k^ and ||H^^-1|| = 1 / lmin of the Jacobi-scaled anchored information"""
        nf = len(self.f)
        if nf == 0:
            self.lmin = self.lmax = self.kappa = 1.0
            return
        s = 1.0 / np.sqrt(self.h)
        Hs = (sp.diags(s) @ self.Hf @ sp.diags(s)).tocsc()
        if nf <= DENSE_EIG_MAX:
            ev = np.linalg.eigvalsh(Hs.toarray())
            self.lmin, self.lmax = float(ev[0]), float(ev[-1])
        else:
            self.lmin = float(spla.eigsh(Hs, k=1, sigma=0.0, which="LM", return_eigenvectors=False, tol=1e-8)[0])
            self.lmax = float(spla.eigsh(Hs, k=1, which="LA", return_eigenvectors=False, tol=1e-4)[0]) * 1.001
        assert self.lmin > 0, (self.case.id, self.lmin)
        self.kappa = self.lmax / self.lmin

    def product(self, X):
        """H_f X in long double, block row by block row (X: long double, free scalars x columns)"""
        b, nc = self.case.b, X.shape[1]
        X3 = X.reshape(self.nfp, b, nc)
        Y = np.empty((self.nfp, b, nc), dtype=LD)
        step = max(1, (1 << 20) // max(nc * b, 1))                    # block rows per pass: bounds the temporaries
        for r0 in range(0, self.nfp, step):
            r1 = min(self.nfp, r0 + step)
            k0, k1 = self.bptr[r0], self.bptr[r1]
            Y[r0:r1] = np.add.reduceat(np.matmul(self.Hb[k0:k1], X3[self.bc[k0:k1]]), self.bptr[r0:r1] - k0, axis=0)
        return Y.reshape(len(self.f), nc)

    def sample(self, k=SAMPLE):
        """poses the device result is checked at: all of them where the reference is dense, else k spread over the graph"""
        n = self.case.n
        if self.dense or n <= k:
            return np.arange(n)
        rng = np.random.default_rng([n, self.case.d, 64])
        fixed = [0, 1, n - 1, self.case.anchor, *self.case.watch]
        return np.unique(np.concatenate([fixed, rng.choice(n, k - len(fixed), replace=False)]))

    def blocks(self, pairs):
        """Sigma[x_i, x_j] for (i, j) in pairs, long double; zero where i or j is the anchor"""
        case, b = self.case, self.case.b
        pairs = [(int(i), int(j)) for i, j in pairs]
        pos = -np.ones(case.n * b, dtype=np.int64)
        pos[self.f] = np.arange(len(self.f))
        out = np.zeros((len(pairs), b, b), dtype=LD)
        if self.dense:
            if self._S is None and len(self.f):
                A = np.zeros((self.nfp, b, self.nfp, b), dtype=LD)
                A[self.br, :, self.bc, :] = self.Hb
                self._S = sc._ld_inverse(A.reshape(len(self.f), len(self.f)))
            for q, (i, j) in enumerate(pairs):
                if case.anchor not in (i, j):
                    out[q] = self._S[np.ix_(pos[i * b:(i + 1) * b], pos[j * b:(j + 1) * b])]
            return out
        cols = sorted({j for i, j in pairs if case.anchor not in (i, j)})
        lu = spla.splu(self.Hf.tocsc())
        for k0 in range(0, len(cols), 64):
            part = cols[k0:k0 + 64]
            E = np.zeros((len(self.f), b * len(part)))
            for q, p in enumerate(part):
                E[pos[p * b:(p + 1) * b], q * b + np.arange(b)] = 1.0
            X = co.refine(lu, self.product, E, lu.solve(E), steps=2)
            for q, p in enumerate(part):
                for k, (i, j) in enumerate(pairs):
                    if j == p and i != case.anchor:
                        out[k] = X[pos[i * b:(i + 1) * b], q * b:(q + 1) * b]
        return out

    def scale(self, i, j):
        """u k^ ||H^^-1|| / sqrt(h_aa h_cc) over block (i, j): the bound without its constant"""
        b = self.case.b
        pos = -np.ones(self.case.n * b, dtype=np.int64)
        pos[self.f] = np.arange(len(self.f))
        hi, hj = self.h[pos[i * b:(i + 1) * b]], self.h[pos[j * b:(j + 1) * b]]
        return U * self.kappa / self.lmin / np.sqrt(np.outer(hi, hj))


def worst_ratio(ref: Reference, got, want, pairs):
    """largest |got - want| / (u k^ ||H^^-1|| / sqrt(h h)) over the blocks of pairs not touching the anchor: must be <= C"""
    worst = 0.0
    for q, (i, j) in enumerate(pairs):
        if ref.case.anchor in (int(i), int(j)):
            continue
        err = np.abs(np.asarray(got[q], dtype=LD) - np.asarray(want[q], dtype=LD)).astype(np.float64)
        worst = max(worst, float(np.max(err / ref.scale(int(i), int(j)))))
    return worst


_refs: Dict[tuple, Reference] = {}


def reference(name: str, d: int) -> Optional[Reference]:
    """the case's Reference, built once per process"""
    if (name, d) not in _refs:
        _refs[(name, d)] = Reference(make_case(name, d))
    return _refs[(name, d)]


def gauss_jordan_inverse(A, block=32):
    """A^-1 by the arithmetic of the device's sweep (dense_inverse.cu) over all pivots, in fp64: per block of `block`
    pivots, k_gj_pivot's unpivoted Gauss-Jordan of the pivot block (Pinv), Rw = Pinv A_k,: and C = A_:,k, then
    A_ij -= C_i Rw_j, A_kj = Rw_j, A_ik = -C_i Pinv and A_kk = Pinv.  The products run in BLAS order, not the kernels'
    FMA chains, so it reproduces the sweep's rounding behaviour, not its bits."""
    A = np.array(A, dtype=np.float64)
    N = A.shape[0]
    for k0 in range(0, N, block):
        kb = slice(k0, min(N, k0 + block))
        P = A[kb, kb].copy()
        for k in range(P.shape[0]):
            inv = 1.0 / P[k, k]
            pik, pkj = P[:, k].copy(), P[k, :].copy()
            P -= np.outer(pik, pkj) * inv
            P[k, :], P[:, k], P[k, k] = pkj * inv, -pik * inv, inv
        Rw = P @ A[kb, :]
        C = A[:, kb].copy()
        A -= C @ Rw
        A[kb, :] = Rw
        A[:, kb] = -C @ P
        A[kb, kb] = P
    return A

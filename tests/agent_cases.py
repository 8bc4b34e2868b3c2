"""Multi-agent setups whose shape reaches the batched kernels' rarely taken branches, and long-double references of what
those kernels compute.  Helper module of test_agent_cases.py (CPU) and test_gpu_agent_kernels.py (GPU); no fixtures.

The dataset partitions give agents of at most a few hundred poses, at most 16 agents per launch and 60 selection rounds,
so the status and momentum kernels never take a second trip of their lane-strided final sum, the selection never ranks
several warps of agents, and the frame alignment never loops over more than one block of candidates.  Each builder below
names the branch it is for; test_agent_cases.py checks from host facts alone that it really reaches it.

The references are taken in long double from the same doubles the kernels receive; the bounds follow structure_cases.py
(a formula evaluated once more on absolute values, times the dot lengths, times u), so they hold for any summation order.
"""
from __future__ import annotations

import math

import numpy as np

import structure_cases as sc
from oracle import dpgo_oracle as orc

# mirrored from dpgo_kernels.cuh / dpgo_capi_agents.cu
STATUS_ROWS = 32             # rows of an agent's Q per status CTA
ACCEL_THREADS = 128          # poses per momentum CTA
SELECT_MAX_AGENTS = 1024     # agents one selection CTA ranks
ALIGN_THREADS = 256          # block of the robust rotation averaging
STATUS_TABLES_MAX = 32       # job tables kept per first agent
STATUS_DOUBLES = 5
U = sc.U
LD = sc.LD
ld = sc.ld


def status_ctas(n):
    return (n + STATUS_ROWS - 1) // STATUS_ROWS


def accel_ctas(n):
    return (n + ACCEL_THREADS - 1) // ACCEL_THREADS


# ---------------------------------------------------------------------------------------------------------------------
# agents
# ---------------------------------------------------------------------------------------------------------------------
# one launch: n = 1, around one warp of rows, a multiple of 32, and past 32 status CTAs (1025 on) and 32 momentum CTAs
SIZES = (1, 31, 32, 33, 1024, 1025, 2049, 4096, 4097, 5000)
ACCEL_SIZES = (1, 33, 129, 4097, 5000)


def small_sizes(count=120, seed=0):
    """>= 100 agents of 1..40 poses in one launch: many jobs, so the CTA -> job binary search runs 7 levels deep"""
    rng = np.random.default_rng(seed)
    s = rng.integers(1, 41, size=count)
    s[:4] = (1, 32, 33, 40)
    return [int(v) for v in s]


class Agent:
    """one agent's problem: a path of n poses (structure_cases.chain), X on the manifold, a random G"""

    def __init__(self, d, r, n, seed):
        rng = np.random.default_rng([seed, d, r, n])
        self.d, self.r, self.n = d, r, n
        edges = sc.edge_set(rng, d, sc.chain(range(n))) if n > 1 else None
        import dpo_b200.posegraph as pg
        self.case = sc.Case(f"path{n}", d, n, edges if edges is not None else pg.EdgeSet.empty(d), "agent")
        self.Q = self.case.Q()
        self.K = sc.pose_K(self.case, d)
        self.X = orc.manifold_project(rng.standard_normal((r, self.case.N)), d)
        self.G = rng.standard_normal((r, self.case.N))


def public_poses(n, kind, seed=0):
    """'all': every pose, in a shuffled slot order; 'spread': the first pose, both sides of every momentum CTA boundary
    and the last pose, in decreasing order; 'none'"""
    if kind == "all":
        return np.random.default_rng([seed, n]).permutation(n).astype(np.int32)
    if kind == "spread":
        p = {0, n - 1, n // 2}
        for b in range(ACCEL_THREADS, n, ACCEL_THREADS):
            p.update((b - 1, b))
        return np.array(sorted(p, reverse=True), dtype=np.int32)
    return np.zeros(0, dtype=np.int32)


# ---------------------------------------------------------------------------------------------------------------------
# status record: <XQ, X>, <X, G>, |P_X(XQ + G)|^2
# ---------------------------------------------------------------------------------------------------------------------
def check_status(rec, a: Agent, X, what, G=None):
    """fields 0-2 of a status record against long-double references of the iterate X (r x N) and G (default a.G)"""
    G = a.G if G is None else G
    count = X.size
    XQ, XQm = sc.product_ref(a.Q, X)
    Xl = ld(X)
    sc.check_scalar(rec[0], np.sum(XQ * Xl), np.sum(XQm * abs(Xl)), a.K, count, f"{what}: <XQ, X>")
    sc.check_scalar(rec[1], np.sum(Xl * ld(G)), np.sum(abs(Xl) * abs(ld(G))), [0], count, f"{what}: <X, G>")
    P, Pm, _, _ = sc.rgrad_ref(a.Q, G, X, a.d)
    e = sc.stage_c(a.K, a.r, a.d) * U * Pm                          # elementwise bound of the gradient
    ref = np.sum(P * P)
    # |g^2 - p^2| <= 2|p| e + e^2 per element, then the sum of `count` squares in any order
    bound = np.sum(2 * abs(P) * e + e * e) + (count + 2) * U * np.sum((abs(P) + e) ** 2)
    assert abs(LD(rec[2]) - ref) <= bound, f"{what}: |rgrad|^2 {rec[2]!r} vs {float(ref)!r}, bound {float(bound):.3e}"


# ---------------------------------------------------------------------------------------------------------------------
# momentum: gamma / alpha recurrence, Y = polar((1 - alpha) X + alpha V), relative change
# ---------------------------------------------------------------------------------------------------------------------
def momentum_gamma(gamma, N):
    """the device recurrence in its operation order; Python floats round as IEEE doubles, so this is bit for bit"""
    q = (4.0 * N) * N
    return (1.0 + math.sqrt(1.0 + q * (gamma * gamma))) / (2.0 * N)


def momentum_alpha(gamma, N):
    return 1.0 / (gamma * N)


def momentum_M(X, V, alpha):
    """(1 - alpha) X + alpha V in long double from the doubles the kernel reads, and its magnitude"""
    c0 = 1.0 - alpha
    return ld(X) * LD(c0) + ld(V) * LD(alpha), abs(ld(X)) * LD(abs(c0)) + abs(ld(V)) * LD(alpha)


def check_polar_step(Yg, M, Mm, d, poses, what):
    """Y tiles of `poses` against polar(M) (rotation block) and M (translation column).

    Rotation block: the float64 polar factor of M rounded, within 128 r u kappa(M) (the bound of test_gpu_pose_numerics
    for the kernel, doubled for numpy's own SVD), plus 3 |dM|_F / sigma_min for the <= 2 u |M| elementwise difference of
    the kernel's fma from M (the polar factor's absolute condition number is below 2 / sigma_min).  A handful of tiles is
    also taken through the 40-digit reference.  Translation: |y - m| <= 2 u |M|."""
    import pose_references as pr
    r = Yg.shape[0]
    Mt, Mmt, Yt = sc.tiles(np.asarray(M, dtype=np.float64), d), sc.tiles(np.asarray(Mm, dtype=np.float64), d), sc.tiles(Yg, d)
    A = np.transpose(Mt[:, poses, :d], (1, 0, 2))                    # (p, r, d)
    Uu, S, Vt = np.linalg.svd(A, full_matrices=False)
    P = Uu @ Vt
    dM = 2 * U * np.sqrt((np.transpose(Mmt[:, poses, :d], (1, 0, 2)) ** 2).sum(axis=(1, 2)))
    tol = 128 * r * U * S[:, 0] / S[:, -1] + 3 * dM / S[:, -1]
    err = np.abs(np.transpose(Yt[:, poses, :d], (1, 0, 2)) - P).max(axis=(1, 2))
    bad = np.flatnonzero(err > tol)
    assert not len(bad), f"{what}: {len(bad)} tiles off polar(M), first pose {poses[bad[0]]}: {err[bad[0]]:.3e} > {tol[bad[0]]:.3e}"
    for i in sorted({0, len(poses) // 2, len(poses) - 1}):
        assert np.abs(Yt[:, poses[i], :d] - pr.polar(A[i])).max() <= tol[i], f"{what}: pose {poses[i]} vs 40 digits"
    et = np.abs(ld(Yt[:, poses, d]) - sc.tiles(M, d)[:, poses, d])
    assert (et <= 2 * U * Mmt[:, poses, d]).all(), f"{what}: translation column"


def relative_change_ref(X, XP, n):
    """sqrt(|X - XP|^2 / n) in long double and its relative bound: the differences round once (2 u on a square), the
    sum of n (d+1) r squares in any order, the division and the square root (which halves the relative error)"""
    D = ld(X) - ld(XP)
    s = np.sum(D * D)
    return np.sqrt(s / n), (X.size / 2 + 4) * U


# ---------------------------------------------------------------------------------------------------------------------
# shared edges and G
# ---------------------------------------------------------------------------------------------------------------------
class SharedEdges:
    """A table for dpgo_agent_set_shared_edges: a hub public pose with >= 300 outgoing and >= 300 incoming shared edges,
    some duplicated exactly (same slot, T and omega) and some sharing a slot, plus edges at the first and last pose."""

    def __init__(self, d, r, n, seed=0, hub=None, per_dir=310, slots=97):
        rng = np.random.default_rng([seed, d, r, n])
        dh = d + 1
        hub = n // 2 if hub is None else hub
        local = [hub] * (2 * per_dir) + [0, 0, n - 1]
        out = [1] * per_dir + [0] * per_dir + [1, 0, 0]
        m = len(local)
        slot = rng.integers(0, slots, size=m)
        Rm = sc.random_rotations(rng, m, d)
        T = np.zeros((m, dh, dh))
        T[:, :d, :d] = Rm
        T[:, :d, d] = rng.standard_normal((m, d))
        T[:, d, d] = 1.0
        w = rng.uniform(0.5, 1.0, m)
        om = np.empty((m, dh))
        om[:, :d] = (w * rng.uniform(1.0, 100.0, m))[:, None]         # kappa and tau differ: om is not uniform
        om[:, d] = w * rng.uniform(0.5, 10.0, m)
        for src, dst in ((3, 4), (3, 5), (per_dir + 7, per_dir + 8)):   # exact duplicates, in both directions
            if dst < m:
                slot[dst], T[dst], om[dst] = slot[src], T[src], om[src]
        order = rng.permutation(m)                                      # directions interleaved in the input
        self.d, self.r, self.n, self.hub, self.slots = d, r, n, hub, slots
        self.local = np.ascontiguousarray(np.asarray(local)[order], dtype=np.int32)
        self.out = np.ascontiguousarray(np.asarray(out)[order], dtype=np.int32)
        self.slot = np.ascontiguousarray(slot[order], dtype=np.int32)
        self.T = np.ascontiguousarray(T[order])
        self.om = np.ascontiguousarray(om[order])
        self.gathered = rng.standard_normal((slots, r, dh))         # tile s: r x (d+1), stored column-major on the device

    def gathered_device_layout(self, gathered=None):
        g = self.gathered if gathered is None else gathered
        return np.ascontiguousarray(np.transpose(g, (0, 2, 1)).reshape(-1))     # per slot: column c, row a at c r + a

    def G_ref(self, gathered=None):
        """G (r x (d+1) n) of the reference's constructGMatrix in long double and the per-element bound
        (d + 3 + edges of the pose) u sum |terms|"""
        g = ld(self.gathered if gathered is None else gathered)
        d, r, n, dh = self.d, self.r, self.n, self.d + 1
        G = np.zeros((r, n, dh), dtype=LD)
        mag = np.zeros((r, n, dh), dtype=LD)
        cnt = np.bincount(self.local, minlength=n)
        for k in range(len(self.local)):
            Xn, T, om = g[self.slot[k]], ld(self.T[k]), ld(self.om[k])
            if self.out[k]:
                L = (Xn * om[None, :]) @ T.T
                Lm = (abs(Xn) * abs(om)[None, :]) @ abs(T).T
            else:
                L = (Xn @ T) * om[None, :]
                Lm = (abs(Xn) @ abs(T)) * abs(om)[None, :]
            G[:, self.local[k]] -= L
            mag[:, self.local[k]] += Lm
        bound = (d + 3 + cnt)[None, :, None] * U * mag
        return G.reshape(r, n * dh), np.asarray(bound, dtype=np.float64).reshape(r, n * dh)


# ---------------------------------------------------------------------------------------------------------------------
# greedy independent-set selection
# ---------------------------------------------------------------------------------------------------------------------
SELECT_KS = (1, 2, 31, 32, 33, 100, 513, 1023, 1024)
GRAPH_KINDS = ("empty", "path", "star", "complete", "random")
SPECIAL_NORMS = (0.0, -0.0, np.nan, np.inf, 5e-324, 2.2250738585072014e-308 / 3, 1.0, 1.0, 2.5, 1e300)


def agent_graph(k, kind, seed=0):
    """(adj_ptr, adj) of a symmetric agent graph without self loops"""
    nb = [set() for _ in range(k)]
    if kind == "path":
        for a in range(k - 1):
            nb[a].add(a + 1), nb[a + 1].add(a)
    elif kind == "star":
        for a in range(1, k):
            nb[0].add(a), nb[a].add(0)
    elif kind == "complete":
        for a in range(k):
            nb[a].update(b for b in range(k) if b != a)
    elif kind == "random":
        rng = np.random.default_rng([seed, k])
        for _ in range(2 * k):
            a, b = (int(v) for v in rng.integers(0, k, 2))
            if a != b:
                nb[a].add(b), nb[b].add(a)
    ptr = np.zeros(k + 1, dtype=np.int32)
    ptr[1:] = np.cumsum([len(s) for s in nb])
    adj = np.array([b for s in nb for b in sorted(s)], dtype=np.int32)
    return ptr, adj


def graph_kind_for(k):
    """the agent graph each k is run with: every kind at least once, complete only where it stays small"""
    return {1: "empty", 2: "path", 31: "complete", 32: "star", 33: "random", 100: "complete", 513: "random",
            1023: "path", 1024: "star"}[k]


def selection_records(k, rounds, seed=0):
    """(rounds, k, STATUS_DOUBLES) records; field 2 mixes random norms with exact ties, +0 and -0, NaN, +inf and
    subnormals, drawn afresh every round"""
    rng = np.random.default_rng([seed, k])
    rec = rng.standard_normal((rounds, k, STATUS_DOUBLES))
    g = rng.uniform(0.0, 4.0, size=(rounds, k))
    pick = rng.random((rounds, k)) < 0.5
    g[pick] = rng.choice(np.array(SPECIAL_NORMS), size=int(pick.sum()))
    rec[:, :, 2] = g
    return rec


def host_select(g, ptr, adj, tie_rule=True, nan_last=True):
    """the selection rule: agents by |rgrad|^2 decreasing (a NaN ranks as -1, below every norm; +inf stays +inf), ties
    to the lower id, each taken unless a neighbour already is.  tie_rule / nan_last = False give the rule without them,
    so that test_agent_cases.py can show the crafted records tell them apart."""
    k = len(g)
    key = [(-1.0 if (nan_last and g[a] != g[a]) else float(g[a])) for a in range(k)]
    if tie_rule:
        order = sorted(range(k), key=lambda a: (-key[a], a))
    else:
        order = sorted(range(k), key=lambda a: (-key[a], -a))           # ties to the higher id instead
    taken = np.zeros(k, dtype=np.uint8)
    for c in order:
        if not any(taken[b] for b in adj[ptr[c]:ptr[c + 1]]):
            taken[c] = 1
    return taken


# ---------------------------------------------------------------------------------------------------------------------
# robust single rotation averaging
# ---------------------------------------------------------------------------------------------------------------------
ROT_MS = (1, 2, 255, 256, 257, 1000, 5000)


def rotation_inputs(d, m, all_inlier=False, seed=0):
    """m rotations: inliers within 0.01 rad of RTrue, and (unless all_inlier, or m <= 2) 40 % outliers at least
    2 cbar (chordal) from RTrue, so that no residual sits near a GNC threshold and summation order cannot flip a weight"""
    import dist_init_oracle as dio
    rng = np.random.default_rng([seed, d, m, int(all_inlier)])
    RTrue = dio.random_rotation(d, rng)
    n_out = 0 if (all_inlier or m <= 2) else (2 * m) // 5
    R = [RTrue @ dio.axis_rotation(d, 0.01 * rng.standard_normal(), rng) for _ in range(m - n_out)]
    while len(R) < m:
        Rc = dio.random_rotation(d, rng)
        if np.linalg.norm(Rc - RTrue) > 2 * dio.CBAR:
            R.append(Rc)
    R = np.array(R)
    return R[rng.permutation(m)]


def gnc_skipped(R, cbar):
    """the reference's mu0 = min(c^2 / (2 max resid - c^2), 1e-5) <= 0: every residual of the unweighted mean is small"""
    Rm = orc.project_to_rotation_group(R.sum(axis=0))
    res = np.sum((Rm[None] - R) ** 2, axis=(1, 2))
    return 2 * res.max() - cbar * cbar <= 0

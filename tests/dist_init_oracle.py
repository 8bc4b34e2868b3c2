"""CPU restatement of the distributed initialisation (test infrastructure, the checker of DistributedPGO(...,
initialization="distributed") and of dpgo_robust_single_rotation_averaging).

The reference's default multi-robot protocol (PGOAgentParameters::multirobot_initialization, ref
include/DPGO/PGOAgent.h:129): every robot runs a chordal initialisation of its private graph in its own frame
(localInitialization, ref src/PGOAgent.cpp:947-962); robot 0 defines the global frame (:182-185); every other robot joins
it when it first hears from an initialised neighbour (updateNeighborPoses -> initializeInGlobalFrame, :369-440), by
GNC-TLS rotation averaging over the frame transforms its shared loop closures give (computeRobustNeighborTransformTwoStage
:290-331, robustSingleRotationAveraging src/DPGO_utils.cpp:567-629) and the mean translation of the inliers
(singleTranslationAveraging :518-535).  Waves: in wave w >= 1 every agent that is not initialised and has a neighbour
initialised before the wave tries those neighbours in increasing id; the first with a non-empty inlier set wins (ref
examples/MultiRobotExample.cpp:245-256; src/PGOAgent.cpp:395-400: an empty inlier set aborts and waits).
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import numpy as np
import scipy.sparse as sp
from scipy.sparse.csgraph import connected_components

from oracle import dpgo_oracle as orc

CBAR = 2.0 * math.sqrt(2.0) * math.sin(0.25)        # angular2ChordalSO3(0.5), ref src/PGOAgent.cpp:316 (~30 degrees)


def gnc_tls_weight(r: float, mu: float, cbar: float) -> float:
    """ref RobustCost::weight, src/DPGO_robust.cpp:49-61."""
    r2 = r * r
    c2 = cbar * cbar
    if r2 >= (mu + 1) / mu * c2:
        return 0.0
    if r2 <= mu / (mu + 1) * c2:
        return 1.0
    return math.sqrt(c2 * mu * (mu + 1) / r2) - mu


def robust_single_rotation_averaging(RVec: np.ndarray, kappa: Optional[np.ndarray] = None, cbar: float = CBAR):
    """ref src/DPGO_utils.cpp:567-629 with the GNC schedule of src/DPGO_robust.cpp:68-103 (mu *= 1.4, 1000 iterations).
    RVec: (m, d, d).  Returns (R, inlier indices, GNC iterations run, weights)."""
    RVec = np.asarray(RVec, dtype=float)
    m = RVec.shape[0]
    k = np.ones(m) if kappa is None else np.asarray(kappa, dtype=float)
    w = np.ones(m)

    def resid(R):
        return k * np.sum((R[None] - RVec) ** 2, axis=(1, 2))

    R = orc.project_to_rotation_group(np.einsum("m,mab->ab", k, RVec))
    c2 = cbar * cbar
    mu = min(c2 / (2 * resid(R).max() - c2), 1e-5)
    iters = 0
    if mu > 0:
        for it in range(1000):
            R = orc.project_to_rotation_group(np.einsum("m,mab->ab", k * w, RVec))
            w = np.array([gnc_tls_weight(math.sqrt(v), mu, cbar) for v in resid(R)])
            iters = it + 1
            if np.all((w < 1e-8) | (w > 1 - 1e-8)):
                break
            mu *= 1.4
    return R, [int(i) for i in np.flatnonzero(w > 1 - 1e-8)], iters, w


def private_graph_connected(n: int, edges: orc.Measurements) -> bool:
    if n <= 1:
        return True
    A = sp.coo_matrix((np.ones(len(edges)), (edges.p1, edges.p2)), shape=(n, n))
    return connected_components(A, directed=False)[0] == 1


def local_initialization(a: int, n: int, odo: orc.Measurements, prv: orc.Measurements) -> np.ndarray:
    """ref src/PGOAgent.cpp:947-962: chordal initialisation of the private graph, local pose 0 is the gauge."""
    priv = orc.Measurements.concat([odo, prv])
    if not private_graph_connected(n, priv):
        raise ValueError(f"agent {a}: the private pose graph (odometry + private loop closures) is not connected")
    if n == 1:
        return np.hstack([np.eye(odo.d), np.zeros((odo.d, 1))])
    return orc.chordal_initialization(priv, n)


def alignment_candidates(a: int, shared: orc.Measurements) -> Dict[int, List[Tuple[int, int]]]:
    """neighbour -> [(public pose j of the neighbour, index of the first shared edge touching it)], j increasing
    (std::map<PoseID> order; findSharedLoopClosureWithNeighbor, ref src/PGOAgent.cpp:922-934)."""
    first: Dict[Tuple[int, int], int] = {}
    for e in range(len(shared)):
        key = (int(shared.r2[e]), int(shared.p2[e])) if shared.r1[e] == a else (int(shared.r1[e]), int(shared.p1[e]))
        first.setdefault(key, e)
    out: Dict[int, List[Tuple[int, int]]] = {}
    for (b, j) in sorted(first):
        out.setdefault(b, []).append((j, first[(b, j)]))
    return out


def candidate_transform(a: int, e: int, shared: orc.Measurements, T_a: np.ndarray, X_bj: np.ndarray,
                        YLift: np.ndarray) -> np.ndarray:
    """ref computeNeighborTransform, src/PGOAgent.cpp:250-288: T_world2_world1 = T_world2_frame2 T_frame1_frame2^-1
    T_world1_frame1^-1 with the neighbour pose YLift^T X_b,j (not projected again: it is exactly YLift T_b,j)."""
    d = shared.d
    dT = orc._homogeneous(shared.subset([e]))[0]
    Tw2f2 = np.eye(d + 1)
    Tw2f2[:d] = YLift.T @ X_bj
    outgoing = shared.r1[e] == a
    Tf1f2 = dT if outgoing else np.linalg.inv(dT)
    i = int(shared.p1[e] if outgoing else shared.p2[e])
    Tw1f1 = np.eye(d + 1)
    Tw1f1[:d] = T_a[:, i * (d + 1):(i + 1) * (d + 1)]
    return Tw2f2 @ np.linalg.inv(Tf1f2) @ np.linalg.inv(Tw1f1)


def apply_transform(Talign: np.ndarray, T: np.ndarray) -> np.ndarray:
    d = Talign.shape[0] - 1
    n = T.shape[1] // (d + 1)
    Tt = T.reshape(d, n, d + 1).copy()
    Tt = np.einsum("pq,qnc->pnc", Talign[:d, :d], Tt)
    Tt[:, :, d] += Talign[:d, d][:, None]
    return Tt.reshape(d, n * (d + 1))


def distributed_initialization(meas: orc.Measurements, n: int, k: int, r: int = 5, owner: Optional[np.ndarray] = None):
    """Returns (T (d x (d+1)n, every agent in the global frame), X = YLift T, per-agent report dicts)."""
    d, dh = meas.d, meas.d + 1
    owner = orc.contiguous_partition(n, k) if owner is None else np.asarray(owner, dtype=np.int64)
    parts, counts, glob = orc.split_measurements(meas, owner, k)
    YLift = orc.fixed_stiefel_variable(d, r)
    T = [local_initialization(a, int(counts[a]), parts[a][0], parts[a][1]) for a in range(k)]
    cands = [alignment_candidates(a, parts[a][2]) for a in range(k)]
    X: List[Optional[np.ndarray]] = [None] * k
    report = [dict(wave=-1, neighbor=-1, candidates=0, inliers=0, iterations=0) for _ in range(k)]
    X[0] = YLift @ T[0]
    report[0]["wave"] = 0
    ready = {0}
    wave = 0
    while len(ready) < k:
        wave += 1
        before = set(ready)
        for a in range(k):
            if a in before:
                continue
            for b in sorted(cands[a]):
                if b not in before:
                    continue
                Ts = np.array([candidate_transform(a, e, parts[a][2], T[a], X[b][:, j * dh:(j + 1) * dh], YLift)
                               for j, e in cands[a][b]])
                R, inl, its, _ = robust_single_rotation_averaging(Ts[:, :d, :d])
                report[a].update(neighbor=b, candidates=len(Ts), inliers=len(inl), iterations=its)
                if inl:
                    Talign = np.eye(dh)
                    Talign[:d, :d] = R
                    Talign[:d, d] = np.sum(Ts[inl, :d, d], axis=0) / len(inl)
                    T[a] = apply_transform(Talign, T[a])
                    X[a] = YLift @ T[a]
                    report[a]["wave"] = wave
                    ready.add(a)
                    break
        if ready == before:
            rest = sorted(set(range(k)) - ready)
            raise RuntimeError(f"distributed initialisation: agents {rest} cannot join the global frame "
                               f"(no initialised neighbour gives a non-empty inlier set)")
    Tg = np.zeros((d, dh * n))
    for a in range(k):
        cols = (glob[a][:, None] * dh + np.arange(dh)[None, :]).ravel()
        Tg[:, cols] = T[a]
    return Tg, YLift @ Tg, report


def random_rotation(d: int, rng: np.random.Generator) -> np.ndarray:
    if d == 2:
        a = rng.uniform(-np.pi, np.pi)
        return np.array([[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]])
    w, x, y, z = rng.standard_normal(4)
    s = math.sqrt(w * w + x * x + y * y + z * z)
    w, x, y, z = w / s, x / s, y / s, z / s
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def axis_rotation(d: int, angle: float, rng: np.random.Generator) -> np.ndarray:
    if d == 2:
        return np.array([[np.cos(angle), -np.sin(angle)], [np.sin(angle), np.cos(angle)]])
    u = rng.standard_normal(3)
    u /= np.linalg.norm(u)
    K = np.array([[0, -u[2], u[1]], [u[2], 0, -u[0]], [-u[1], u[0], 0]])
    return np.eye(3) + np.sin(angle) * K + (1 - np.cos(angle)) * (K @ K)


def rotation_fixture(d: int, seed: int, inliers: int = 10, outliers: int = 40, cbar: float = None,
                     noise: float = 0.01, near: bool = False) -> Tuple[np.ndarray, float]:
    """Recipe of ref tests/testUtils.cpp:90-118: `inliers` rotations near RTrue (angle noise `noise` rad), then random
    outliers farther than 1.2 cbar from RTrue (cbar = angular2ChordalSO3(0.3)).  near: half of the outliers sit just
    beyond the threshold (chordal distance 1.0-1.3 cbar), so residuals cross the GNC bounds late."""
    rng = np.random.default_rng(seed)
    cbar = 2 * math.sqrt(2) * math.sin(0.15) if cbar is None else cbar
    RTrue = random_rotation(d, rng)
    RVec = [RTrue @ axis_rotation(d, noise * rng.standard_normal(), rng) for _ in range(inliers)]
    while len(RVec) < inliers + outliers:
        if near and len(RVec) % 2 == 0:
            chord = cbar * rng.uniform(1.0, 1.3)
            R = RTrue @ axis_rotation(d, 2 * math.asin(min(1.0, chord / (2 * math.sqrt(2)))), rng)   # |R(a) - I|_F
            RVec.append(R)
            continue
        R = random_rotation(d, rng)
        if np.linalg.norm(R - RTrue) > 1.2 * cbar:
            RVec.append(R)
    return np.array(RVec), cbar

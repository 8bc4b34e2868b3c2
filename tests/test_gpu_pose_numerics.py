"""The per-pose kernels on crafted tiles against 40-digit references (pose_references.py): the Stiefel projection
(k_stiefel_project), the projection onto SO(d) (project_to_rotation, shared by the chordal start, the frame alignment and
the rounded trajectory; reached here through dpgo_agent_trajectory_global) and the QF retraction.  Crafted tiles: graded,
widely spread and repeated singular values, orthonormal tiles, det < 0, scales 1e+-100 and exactly rank-deficient tiles."""
import numpy as np
import pytest

import pose_references as pr
import structure_cases as sc
from oracle import dpgo_oracle as orc

pytestmark = pytest.mark.gpu

DR = [(d, r) for d in (2, 3) for r in sc.RANKS[d]]
U = sc.U


def problem(n, d, r):
    """a chain of n poses (the retraction runs in the persistent kernel, which needs rows to own)"""
    import dpo_b200 as dp
    c = sc.Case("chain", d, n, sc.edge_set(np.random.default_rng(0), d, sc.chain(range(n))), "")
    gp = dp.QuadraticProblem(n, d, r, preconditioners=(dp.PRECOND_BLOCK_JACOBI,))
    gp.setQ(c.Q())
    return gp


def pack(mats, d, r, rng):
    """tiles [M | t] side by side, M padded below to r rows with the rows given (r x d), t random"""
    X = np.zeros((r, (d + 1) * len(mats)))
    for i, M in enumerate(mats):
        X[:, i * (d + 1):i * (d + 1) + d] = M
        X[:, i * (d + 1) + d] = rng.standard_normal(r)
    return X


@pytest.mark.parametrize("d,r", DR)
def test_stiefel_projection(d, r):
    rng = np.random.default_rng([d, r])
    tiles = pr.crafted_tiles(rng, r, d)
    X = pack([M for _, M, _ in tiles], d, r, rng)
    gp = problem(len(tiles), d, r)
    Y = gp.project(X)
    for i, (label, M, unique) in enumerate(tiles):
        Yi = Y[:, i * (d + 1):i * (d + 1) + d]
        what = (label, i)
        assert np.abs(Yi.T @ Yi - np.eye(d)).max() <= 8 * r * U, what
        _, S, _ = pr.svd(M)
        assert abs(np.sum(Yi * M) - S.sum()) <= 8 * r * d * U * S.sum() + 1e-300, what     # the polar factor maximises <Y, M>
        if unique:
            assert np.abs(Yi - pr.polar(M)).max() <= 64 * r * U * S[0] / S[-1], what
        if r == d and label == "det_neg":
            assert abs(np.linalg.det(Yi) + 1.0) <= 1e-13, what
        assert np.array_equal(Y[:, i * (d + 1) + d], X[:, i * (d + 1) + d]), what


@pytest.mark.parametrize("d,r", DR)
def test_rotation_projection(d, r):
    """T_i = [proj_SO(d)(Ya^T Y_i) | Ya^T p_i - Ya^T pa] with the anchor Ya = [e_1 .. e_d], pa = 0: the top d x d block of
    each tile goes through project_to_rotation unchanged"""
    from dpo_b200 import _capi as capi
    rng = np.random.default_rng([d, r, 1])
    tiles = pr.crafted_tiles(rng, d, d)
    mats = [np.vstack([M, rng.standard_normal((r - d, d))]) for _, M, _ in tiles]
    X = pack(mats, d, r, rng)
    gp = problem(len(tiles), d, r)
    gp.upload_X(X)
    anchor = np.zeros((r, d + 1), order="F")
    anchor[:d, :d] = np.eye(d)
    out = np.zeros((d, (d + 1) * len(tiles)), order="F")
    capi.check(gp._lib.dpgo_agent_trajectory_global(gp._h, capi.dptr(anchor), capi.dptr(out)))
    for i, (label, M, _) in enumerate(tiles):
        R = out[:, i * (d + 1):i * (d + 1) + d]
        what = (label, i)
        # all singular values 1: every Jacobi rotation is driven by rounding noise and turns the basis by an arbitrary
        # angle, each adding its own rounding (30 u measured at d = 3 on the draw of r = 8)
        assert np.abs(R.T @ R - np.eye(d)).max() <= (16 if label == "sv_ones" else 8) * d * U, what
        assert abs(np.linalg.det(R) - 1.0) <= 1e-13, what
        Rref = pr.rotation(M)
        _, S, _ = pr.svd(M)
        assert np.linalg.norm(R - M) <= np.linalg.norm(Rref - M) + 64 * d * U * max(S[0], 1.0), what     # the optimum
        # the minimiser is unique unless the two smallest singular values tie (det < 0) or sum to zero (det >= 0)
        gap = (S[-2] - S[-1]) if np.linalg.det(M) < 0 else (S[-2] + S[-1])
        if S[0] > 0 and gap > 1e-6 * S[0]:
            assert np.abs(R - Rref).max() <= 64 * d * U * S[0] / gap, what
        assert np.array_equal(out[:, i * (d + 1) + d], X[:d, i * (d + 1) + d]), what


@pytest.mark.parametrize("d,r", DR)
def test_qf_retraction(d, r):
    rng = np.random.default_rng([d, r, 2])
    Xs, Es = [], []
    for k in (1.0, 1e2, 1e4, 1e6, 1e8):
        for _ in range(2):
            Xi = np.linalg.qr(rng.standard_normal((r, d)))[0]
            W = pr.with_singular_values(rng, r, d, np.geomspace(1.0, 1.0 / k, d))
            Xs.append(Xi)
            Es.append(W - Xi)
    for _ in range(2):
        Xi = np.linalg.qr(rng.standard_normal((r, d)))[0]
        E = rng.standard_normal((r, d))
        Xs.append(Xi)
        Es.append(1e4 * E / np.linalg.norm(E))
        Xs.append(Xi)
        Es.append(np.zeros((r, d)))
    X = pack(Xs, d, r, rng)
    eta = pack(Es, d, r, rng)
    gp = problem(len(Xs), d, r)
    out = gp.Retraction(X, eta)
    W = X + eta
    for i in range(len(Xs)):
        Wi = W[:, i * (d + 1):i * (d + 1) + d]
        Qi = out[:, i * (d + 1):i * (d + 1) + d]
        _, S, _ = pr.svd(Wi)
        assert np.abs(Qi.T @ Qi - np.eye(d)).max() <= 16 * r * U, i
        assert np.abs(Qi - pr.qf(Wi)).max() <= 64 * r * U * S[0] / S[-1], i
        assert np.array_equal(out[:, i * (d + 1) + d], W[:, i * (d + 1) + d]), i
    assert np.abs(out - orc.retract(X, eta, d)).max() <= 1e-6           # the oracle's numpy QR, for orientation

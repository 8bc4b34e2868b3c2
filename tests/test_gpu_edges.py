"""Device-side Q assembly from raw edge records and robust re-weighting (SURVEY 8f rank 2): k_assemble_Q against the host
construction (ref constructConnectionLaplacianSE, src/DPGO_utils.cpp:199-271), k_edge_weights against the reference's
scalar formulas (computeMeasurementError :494-500, RobustCost::weight src/DPGO_robust.cpp:23-66)."""
import os

import numpy as np
import pytest

from oracle import dpgo_oracle as orc

pytestmark = pytest.mark.gpu


def relerr(a, b):
    return float(np.linalg.norm(np.asarray(a) - np.asarray(b)) / max(np.linalg.norm(b), 1e-300))


def host_weight(cost, r, mu, c):
    if cost == "L2":
        return 1.0
    if cost == "L1":
        return 1.0 / r
    if cost == "Huber":
        return 1.0 if r < c else c / r
    if cost == "TLS":
        return 1.0 if r < c else 0.0
    if cost == "GM":
        return 1.0 / (1.0 + r * r) ** 2
    r2, c2 = r * r, c * c
    if r2 >= (mu + 1) / mu * c2:
        return 0.0
    if r2 <= mu / (mu + 1) * c2:
        return 1.0
    return np.sqrt(c2 * mu * (mu + 1) / r2) - mu


@pytest.mark.parametrize("ds,r", [("smallGrid3D", 5), ("sphere2500", 5), ("CSAIL", 3), ("tinyGrid3D", 3)])
def test_device_assembly_and_reweighting(ds, r, data_dir):
    import dpo_b200 as dp
    from dpo_b200 import posegraph as pg
    edges, n = pg.read_g2o_file(os.path.join(data_dir, ds + ".g2o"))
    meas, _ = orc.read_g2o(os.path.join(data_dir, ds + ".g2o"))
    d, dh = edges.d, edges.d + 1
    rng = np.random.default_rng(11)
    X = orc.manifold_project(rng.standard_normal((r, dh * n)), d)
    V = rng.standard_normal(X.shape)
    # ---- assembly with non-trivial initial weights ----
    w0 = rng.uniform(0.2, 1.0, len(edges))
    edges.weight = w0.copy()
    meas.weight = w0.copy()
    gp = dp.QuadraticProblem(n, d, r)
    fixed = (edges.p1 + 1 == edges.p2).astype(np.int32)                    # odometry keeps its weight
    gp.setEdges(edges, fixed=fixed)
    op = orc.QuadraticProblem(n, d, r)
    op.set_Q(orc.construct_connection_laplacian(meas, n))
    assert abs(gp.f(X) - op.f(X)) <= 1e-12 * abs(op.f(X))
    assert relerr(gp.EucGrad(X), op.euc_grad(X)) <= 1e-13
    assert relerr(gp.PreConditioner(X, V), op.precondition(X, V)) <= 1e-10    # preconditioners follow the device-built Q
    # ---- robust re-weighting at the resident iterate, every loss ----
    T = np.zeros((len(edges), dh, dh)); T[:, :d, :d] = edges.R; T[:, :d, d] = edges.t; T[:, d, d] = 1
    Xt = X.reshape(r, n, dh, order="F") if False else np.stack([X[:, p * dh:(p + 1) * dh] for p in range(n)])      # (n, r, dh)
    Y1, Y2 = Xt[edges.p1][:, :, :d], Xt[edges.p2][:, :, :d]
    q1, q2 = Xt[edges.p1][:, :, d], Xt[edges.p2][:, :, d]
    rot = np.sum((np.einsum("mab,mbc->mac", Y1, edges.R) - Y2) ** 2, axis=(1, 2))
    tra = np.sum((q2 - q1 - np.einsum("mab,mb->ma", Y1, edges.t)) ** 2, axis=1)
    r2_ref = edges.kappa * rot + edges.tau * tra                              # ref computeMeasurementError
    for cost, mu, c in (("GNC_TLS", 0.05, 3.0), ("GNC_TLS", 2.0, 1.5), ("Huber", 1.0, 2.0), ("TLS", 1.0, 2.5), ("GM", 1.0, 1.0),
                        ("L1", 1.0, 1.0), ("L2", 1.0, 1.0)):
        gp.setEdgeWeights(w0)
        gp.upload_X(X)
        w, r2 = gp.robustReweight(cost, mu=mu, param=c)
        assert np.max(np.abs(r2 - r2_ref) / np.maximum(r2_ref, 1e-300)) <= 1e-11
        w_ref = np.array([w0[e] if fixed[e] else host_weight(cost, np.sqrt(r2_ref[e]), mu, c) for e in range(len(edges))])
        assert np.max(np.abs(w - w_ref)) <= 1e-9 * max(1.0, np.max(np.abs(w_ref))), cost
        meas.weight = w_ref.copy()
        op.set_Q(orc.construct_connection_laplacian(meas, n))
        assert relerr(gp.EucGrad(X), op.euc_grad(X)) <= 1e-11, cost
        if cost in ("GNC_TLS", "Huber"):
            assert relerr(gp.PreConditioner(X, V), op.precondition(X, V)) <= 1e-9, cost   # exact preconditioner rebuilt for the new Q

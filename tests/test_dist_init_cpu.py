"""Distributed initialisation without a GPU: the oracle's GNC-TLS rotation averaging against the C++ host restatement in
libDPGO (ref robustSingleRotationAveraging, src/DPGO_utils.cpp:567-629), the oracle's wave driver on a noise-free lattice
(known answer: ground truth in agent 0's gauge), the host-side candidate tables, and the error paths."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import dist_init_oracle as dio  # noqa: E402
from dpo_b200 import posegraph as pg  # noqa: E402
from oracle import dpgo_oracle as orc  # noqa: E402


def to_meas(edges):
    return orc.Measurements(edges.d, edges.r1, edges.r2, edges.p1, edges.p2, edges.R, edges.t, edges.kappa, edges.tau,
                            edges.weight)


@pytest.fixture(scope="module")
def averaging_check():
    from dpo_b200 import build
    return build.build_cpp_program([os.path.join(ROOT, "tests", "cpp", "robust_averaging_check.cpp")],
                                   os.path.join(ROOT, "build", "tests", "robust_averaging_check"))


def host_average(exe, RVec, cbar, tmp_path):
    path = tmp_path / "fixture.txt"
    m, d = RVec.shape[0], RVec.shape[1]
    with open(path, "w") as fh:
        fh.write(f"{d} {m} {cbar!r}\n")
        for R in RVec:
            fh.write(" ".join(repr(float(v)) for v in R.ravel()) + "\n")
    res = subprocess.run([exe, str(path)], capture_output=True, text=True, timeout=60)
    assert res.returncode == 0, res.stderr[-2000:]
    rec = {ln.split()[0]: ln.split()[1:] for ln in res.stdout.splitlines() if ln.strip()}
    return np.array([float(v) for v in rec["R"]]).reshape(d, d), [int(v) for v in rec.get("inliers", [])]


@pytest.mark.parametrize("d,outliers", [(3, 40), (2, 15)])
@pytest.mark.parametrize("seed", range(6))
def test_robust_rotation_averaging_matches_host(averaging_check, d, outliers, seed, tmp_path):
    """ref tests/testUtils.cpp:90-118 recipe: 10 noisy inliers and random outliers farther than 1.2 cbar; both sides find
    exactly the 10.  SO(2) runs with 15 outliers: see the test below for 40."""
    RVec, cbar = dio.rotation_fixture(d, seed, outliers=outliers)
    R, inl, its, _ = dio.robust_single_rotation_averaging(RVec, cbar=cbar)
    Rh, inl_h = host_average(averaging_check, RVec, cbar, tmp_path)
    assert inl == inl_h == list(range(10))
    assert np.abs(R - Rh).max() <= 1e-12
    assert its > 0


def test_so2_forty_outliers_agree_with_host(averaging_check, tmp_path):
    """With the recipe's 40 outliers, SO(2) is different from SO(3): on the circle the 40 outliers leave about
    40 * 0.6 / (2 pi) ~ 4 of them inside any threshold-wide window, and GNC, which starts from the all-weights mean, ends in a
    spurious basin for a good part of the seeds (16 of seeds 0-29 recover exactly the 10).  That is the algorithm, not the
    restatement: the host's C++ restatement returns the same inlier set and rotation on every seed."""
    recovered = 0
    for seed in range(12):
        RVec, cbar = dio.rotation_fixture(2, seed)
        R, inl, _, _ = dio.robust_single_rotation_averaging(RVec, cbar=cbar)
        Rh, inl_h = host_average(averaging_check, RVec, cbar, tmp_path)
        assert inl == inl_h and np.abs(R - Rh).max() <= 1e-12
        recovered += inl == list(range(10))
    assert 0 < recovered < 12


@pytest.mark.parametrize("d", [2, 3])
def test_robust_rotation_averaging_trivial(averaging_check, d, tmp_path):
    """ref tests/testUtils.cpp:72-88: one measurement (and here also several identical ones): every residual is zero,
    mu0 <= 0 and GNC is skipped."""
    rng = np.random.default_rng(7)
    RTrue = dio.random_rotation(d, rng)
    for m in (1, 5):
        RVec = np.array([RTrue] * m)
        R, inl, its, _ = dio.robust_single_rotation_averaging(RVec)
        Rh, inl_h = host_average(averaging_check, RVec, dio.CBAR, tmp_path)
        assert its == 0 and inl == inl_h == list(range(m))
        assert np.abs(R - Rh).max() <= 1e-12 and np.abs(R - RTrue).max() <= 1e-12


def test_known_answer_noise_free_lattice():
    """Noise-free 16 x 16 x 4 lattice in 8 blocks: every agent's local chordal start is exact in its own frame, so the
    distributed start is the ground truth expressed in the frame of agent 0's first pose."""
    nx, ny, nz, k = 16, 16, 4, 8
    edges, n, Tgt = pg.synthetic_grid_graph(nx, ny, nz, edges_per_pose=3.5, seed=4, rot_sigma=0.0, trans_sigma=0.0)
    owner = pg.grid_block_owner(nx, ny, nz, k)
    T, X, report = dio.distributed_initialization(to_meas(edges), n, k, owner=owner)
    g0 = int(np.flatnonzero(owner == 0)[0])
    H = np.eye(4)
    H[:3] = Tgt[:, 4 * g0:4 * g0 + 4]
    expected = dio.apply_transform(np.linalg.inv(H), Tgt)
    assert np.abs(T - expected).max() <= 1e-9
    assert np.allclose(X, orc.fixed_stiefel_variable(3, 5) @ T, rtol=0, atol=1e-12)
    assert report[0]["wave"] == 0 and all(rep["wave"] >= 1 and rep["inliers"] == rep["candidates"] for rep in report[1:])


def test_candidate_tables_match_oracle():
    """The product's host table (dpgo_agent_set_align_candidates input) lists the oracle's candidates in its order."""
    from dpo_b200.agent import ExchangePlan, alignment_candidates, contiguous_owner, partition_edges
    edges, n = pg.read_g2o_file(os.path.join(ROOT, "data", "torus3D.g2o"))
    meas, _ = orc.read_g2o(os.path.join(ROOT, "data", "torus3D.g2o"))
    k = 8
    parts, _, _ = partition_edges(edges, contiguous_owner(n, k), k)
    plan = ExchangePlan([p[2] for p in parts], k)
    oparts, _, _ = orc.split_measurements(meas, orc.contiguous_partition(n, k), k)
    for a in range(k):
        ct = alignment_candidates(a, parts[a][2], plan)
        oc = dio.alignment_candidates(a, oparts[a][2])
        assert list(ct["neighbor"]) == sorted(oc)
        flat = [(b, j, e) for b in sorted(oc) for j, e in oc[b]]
        assert list(np.diff(ct["ptr"])) == [len(oc[b]) for b in sorted(oc)]
        assert list(ct["slot"]) == [plan.slot(b, j) for b, j, _ in flat]
        sh = oparts[a][2]
        assert list(ct["local"]) == [int(sh.p1[e] if sh.r1[e] == a else sh.p2[e]) for _, _, e in flat]
        assert list(ct["outgoing"]) == [int(sh.r1[e] == a) for _, _, e in flat]


def _split_slabs():
    """8 x 2 x 2 lattice cut into four 2-wide slabs along x; agent 1 owns slabs 1 and 3, which do not touch."""
    edges, n, _ = pg.synthetic_grid_graph(8, 2, 2, edges_per_pose=1.0, seed=0)
    slab = pg.grid_lattice_coords(8, 2, 2)[:, 0] // 2
    return edges, n, np.array([0, 1, 2, 1])[slab]


def test_disconnected_private_graph_names_the_agent():
    from dpo_b200.agent import check_private_graph_connected, partition_edges
    from dpo_b200.posegraph import EdgeSet
    edges, n, owner = _split_slabs()
    with pytest.raises(ValueError, match="agent 1"):
        dio.distributed_initialization(to_meas(edges), n, 3, owner=owner)
    parts, counts, _ = partition_edges(edges, owner, 3)
    check_private_graph_connected(0, int(counts[0]), EdgeSet.join([parts[0][0], parts[0][1]]))
    with pytest.raises(ValueError, match="agent 1"):
        check_private_graph_connected(1, int(counts[1]), EdgeSet.join([parts[1][0], parts[1][1]]))


def disconnect_last_agent(meas, n, k):
    """Drop every edge between the last agent of the contiguous split and the others: a disconnected agent graph."""
    owner = orc.contiguous_partition(n, k)
    a1, a2 = owner[meas.p1], owner[meas.p2]
    keep = ~((a1 != a2) & ((a1 == k - 1) | (a2 == k - 1)))
    return meas.subset(np.flatnonzero(keep))


def test_disconnected_agent_graph_names_the_agent():
    meas, n = orc.read_g2o(os.path.join(ROOT, "data", "smallGrid3D.g2o"))
    with pytest.raises(RuntimeError, match=r"agents \[3\]"):
        dio.distributed_initialization(disconnect_last_agent(meas, n, 4), n, 4)

"""Pose marginal covariances on the GPU (dpgo_pose_covariances / pg.poseCovariancesGPU) against the NumPy/SciPy
restatement of the model (covariance_oracle): per-pose blocks, pair blocks, anchors, weights, repeatability, argument
checks, and the runner's pose_covariances()."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import covariance_oracle as co  # noqa: E402
from dpo_b200 import posegraph as pg  # noqa: E402

pytestmark = pytest.mark.gpu

DATA = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "data")
_cache = {}


def problem(name):
    """The dataset and the oracle's chordal initialisation (a rounded trajectory)."""
    if name not in _cache:
        edges, n = pg.read_g2o_file(os.path.join(DATA, name + ".g2o"))
        _cache[name] = (edges, n, pg.chordalInitialization(edges.d, n, edges))
    return _cache[name]


def rel(a, b):
    return np.linalg.norm(a - b) / np.linalg.norm(b)


def check_blocks(cov, want, poses, anchor, tol=1e-9):
    for k, p in enumerate(poses):
        if p == anchor:
            assert np.all(cov[p] == 0)
            continue
        assert rel(cov[p], want[k]) <= tol, (p, rel(cov[p], want[k]))
        assert np.array_equal(cov[p], cov[p].T)
        assert np.linalg.eigvalsh(cov[p])[0] > 0


@pytest.mark.parametrize("name", ["tinyGrid3D", "smallGrid3D", "input_INTEL_g2o", "sphere2500"])
def test_every_pose_matches_the_dense_oracle(name):
    edges, n, T = problem(name)
    b = co.tangent_dim(edges.d)
    cov = pg.poseCovariancesGPU(edges, n, T)
    S = co.covariances_dense(co.information(T, edges, n), n, b, 0)
    check_blocks(cov, co.blocks_of(S, b, [(p, p) for p in range(n)]), range(n), 0)


# The oracle's columns are refined with extended-precision residuals, so they are accurate well beyond fp64 factorisations.
# ais2klinik's anchored information is far worse conditioned than the others (its covariance blocks span 1e-2 .. 1e4):
# there an unrefined splu is 1.1e-8 and the host emulation's Cholesky factorisation 1.2e-7 away from the refined oracle
# on the worst of these 64 blocks, so no fp64 factorisation without refinement meets 1e-9 on it; its bound is 3e-7
@pytest.mark.parametrize("name,tol", [("torus3D", 1e-9), ("grid3D", 1e-9), ("city10000", 1e-9), ("ais2klinik", 3e-7)])
def test_sampled_poses_match_splu(name, tol):
    edges, n, T = problem(name)
    b = co.tangent_dim(edges.d)
    cov, info = pg.poseCovariancesGPU(edges, n, T, return_info=True)
    sample = np.random.default_rng(64).choice(np.arange(1, n), 64, replace=False)
    want = co.block_sample(co.information(T, edges, n), n, b, 0, [(p, p) for p in sample])
    check_blocks(cov, want, sample, 0, tol)
    assert np.all(cov[0] == 0)
    assert all(np.array_equal(c, c.T) for c in cov)
    assert info[0] >= 1 and info[2] == n * b // 3 and info[11] > 0


def test_pair_blocks_inside_and_across_fronts():
    edges, n, T = problem("smallGrid3D")
    b = 6
    rng = np.random.default_rng(3)
    near = np.stack([edges.p1[:8], edges.p2[:8]], 1)                 # measured pairs: adjacent in the pattern already
    far = np.stack([rng.choice(n, 2, replace=False) for _ in range(12)])   # mostly in unrelated subtrees
    pairs = np.concatenate([near, far, [[5, 5], [0, 9], [9, 0]]])
    cov, pcov = pg.poseCovariancesGPU(edges, n, T, pairs=pairs)
    S = co.covariances_dense(co.information(T, edges, n), n, b, 0)
    want = co.blocks_of(S, b, pairs)
    for k, (i, j) in enumerate(pairs):
        if i == 0 or j == 0:
            assert np.all(pcov[k] == 0)
        else:
            assert rel(pcov[k], want[k]) <= 1e-9, (i, j)
    assert np.array_equal(pcov[-3], cov[5])
    base = pg.poseCovariancesGPU(edges, n, T)
    check_blocks(base, co.blocks_of(S, b, [(p, p) for p in range(n)]), range(n), 0)


def test_two_calls_are_bitwise_equal_and_the_anchor_moves():
    edges, n, T = problem("input_INTEL_g2o")
    a = pg.poseCovariancesGPU(edges, n, T, anchor=0)
    b_ = pg.poseCovariancesGPU(edges, n, T, anchor=0)
    assert np.array_equal(a, b_)
    anchor = 611
    c = pg.poseCovariancesGPU(edges, n, T, anchor=anchor)
    S = co.covariances_dense(co.information(T, edges, n), n, 3, anchor)
    check_blocks(c, co.blocks_of(S, 3, [(p, p) for p in range(n)]), range(n), anchor)


def test_weights_are_honoured():
    edges, n, T = problem("smallGrid3D")
    w = np.random.default_rng(11).uniform(0.05, 2.0, len(edges))
    we = pg.EdgeSet(edges.d, edges.r1, edges.r2, edges.p1, edges.p2, edges.R, edges.t, edges.kappa, edges.tau, weight=w)
    cov = pg.poseCovariancesGPU(we, n, T)
    S = co.covariances_dense(co.information(T, we, n), n, 6, 0)
    check_blocks(cov, co.blocks_of(S, 6, [(p, p) for p in range(n)]), range(n), 0)
    assert rel(cov[1:], pg.poseCovariancesGPU(edges, n, T)[1:]) > 1e-3


def test_device_agrees_with_the_host_emulation():
    from dpo_b200 import _capi as capi
    lib = capi.load_library()
    edges, n, T = problem("smallGrid3D")
    p1, p2, R, t, kappa, tau, w = co.edge_arrays(edges)
    host = np.zeros((n, 6, 6))
    Tf = np.asfortranarray(T)
    capi.check(lib.dpgo_pose_covariances_debug_emulate(n, 3, len(p1), capi.iptr(p1), capi.iptr(p2), capi.dptr(R), capi.dptr(t),
                                                       capi.dptr(kappa), capi.dptr(tau), capi.dptr(w), capi.dptr(Tf), 0, -1, 0,
                                                       0, None, capi.dptr(host), None, None))
    assert rel(pg.poseCovariancesGPU(edges, n, T), host) <= 1e-11


def call(n, d, edges, T, anchor=0, pairs=None):
    from dpo_b200 import _capi as capi
    lib = capi.load_library()
    p1, p2, R, t, kappa, tau, w = co.edge_arrays(edges)
    b = 6 if d == 3 else 3
    pr = np.zeros((0, 2), np.int32) if pairs is None else np.ascontiguousarray(np.asarray(pairs, np.int32))
    cov = np.zeros((max(n, 1), b, b))
    pc = np.zeros((max(len(pr), 1), b, b))
    Tp = None if T is None else capi.dptr(np.asfortranarray(T))
    code = lib.dpgo_pose_covariances(n, d, len(p1), capi.iptr(p1), capi.iptr(p2), capi.dptr(R), capi.dptr(t), capi.dptr(kappa),
                                     capi.dptr(tau), capi.dptr(w), Tp, anchor, 0, len(pr), capi.iptr(pr), capi.dptr(cov),
                                     capi.dptr(pc), None)
    return code, capi.last_error()


def test_invalid_arguments_are_refused():
    edges, n, T = problem("tinyGrid3D")
    assert call(n, 3, edges, T, anchor=n)[0] == 1
    assert call(n, 3, edges, T, anchor=-1)[0] == 1
    assert call(n, 3, edges, T, pairs=[[0, n]])[0] == 1
    bad = edges.take(np.arange(len(edges)))
    bad.p2 = bad.p2.copy()
    bad.p2[3] = n + 4
    assert call(n, 3, bad, T)[0] == 1
    assert call(n, 4, edges, T)[0] == 1
    code, msg = call(n, 3, edges, None)
    assert code == 1 and "null" in msg
    with pytest.raises(ValueError):
        pg.poseCovariancesGPU(edges, n, T[:, :-4])


def test_a_disconnected_graph_is_an_error():
    edges, n, T = problem("tinyGrid3D")
    last = n - 1
    keep = np.nonzero((edges.p1 != last) & (edges.p2 != last))[0]
    code, msg = call(n, 3, edges.take(keep), T)
    assert code == 1 and "not connected" in msg


def test_runner_pose_covariances_is_the_function_on_its_trajectory():
    from dpo_b200.agent import DistributedPGO
    edges, n, _ = problem("smallGrid3D")
    run = DistributedPGO(edges, n, 4, r=5, schedule="coloured")
    run.solve(max_rounds=30)
    T = run.trajectory()
    want = pg.poseCovariancesGPU(edges, n, T)
    got = run.pose_covariances()
    assert np.array_equal(got, want)


def test_a_singular_information_fails_in_the_factorisation():
    """Every edge of one pose has tau = 0: the graph is connected (kappa > 0), so the argument check passes, but the
    pose's translation is free and its pivot is exactly 0.  Reported as DPGO_ERR_CUDA, not as numbers."""
    edges, n, T = problem("tinyGrid3D")
    p = 7
    e = edges.take(np.arange(len(edges)))
    e.tau = np.where((e.p1 == p) | (e.p2 == p), 0.0, e.tau)
    code, msg = call(n, 3, e, T)
    assert code == 3 and "not positive definite" in msg, (code, msg)
    assert call(n, 3, edges, T)[0] == 0                 # the same graph with its tau values: no error


def _sanitizer():
    import shutil
    for c in (shutil.which("compute-sanitizer"), "/usr/local/cuda/bin/compute-sanitizer"):
        if c and os.path.exists(c):
            return c
    return None


def test_memcheck_of_small_calls_reports_no_errors(tmp_path):
    """compute-sanitizer memcheck over one SE(3) call with pairs and one SE(2) call (tests/_covariance_sanitizer_worker.py):
    every read and write of the assembly, factorisation and sweep kernels stays inside its buffers."""
    import subprocess
    tool = _sanitizer()
    if tool is None:
        pytest.skip("compute-sanitizer is not installed")
    worker = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_covariance_sanitizer_worker.py")
    res = subprocess.run([tool, "--tool", "memcheck", "--leak-check", "no", sys.executable, worker], capture_output=True,
                         text=True, timeout=900)
    out = res.stdout + res.stderr
    if "Device not supported" in out or "ERROR SUMMARY" not in out:
        pytest.skip("compute-sanitizer cannot check this device or could not start its target: " + out[:300])
    assert "ERROR SUMMARY: 0 errors" in out and res.returncode == 0, out[-3000:]
    assert "ok" in res.stdout


@pytest.fixture(scope="module")
def covariance_check():
    from dpo_b200 import build
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    return build.build_cpp_program([os.path.join(root, "tests", "cpp", "covariance_check.cpp")],
                                   os.path.join(root, "build", "tests", "covariance_check"))


def test_cpp_device_rbcd_pose_covariances_match_python(covariance_check, tmp_path):
    """DeviceRBCD::poseCovariances (C++) equals pg.poseCovariancesGPU (Python) called on the C++ runner's trajectory, for the
    pose blocks and for requested pairs.  The readers compute kappa / tau each in their own arithmetic, so the bound is
    1e-12 rather than bit equality."""
    import subprocess
    edges, n, _ = problem("smallGrid3D")
    pairs = [(3, 40), (10, 11), (0, 7)]
    res = subprocess.run([covariance_check, os.path.join(DATA, "smallGrid3D.g2o"), "4", "20", str(tmp_path)] +
                         [str(v) for pq in pairs for v in pq], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-2000:]
    T = np.loadtxt(os.path.join(str(tmp_path), "trajectory.txt"))
    cov_c = np.loadtxt(os.path.join(str(tmp_path), "cov.txt")).reshape(n, 6, 6)
    pc_c = np.loadtxt(os.path.join(str(tmp_path), "pairs.txt")).reshape(len(pairs), 6, 6)
    cov_p, pc_p = pg.poseCovariancesGPU(edges, n, T, pairs=pairs)
    assert rel(cov_c, cov_p) <= 1e-12 and rel(pc_c, pc_p) <= 1e-12
    assert np.all(cov_c[0] == 0) and np.all(pc_c[2] == 0)

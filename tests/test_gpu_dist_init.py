"""Distributed initialisation on the GPU (DistributedPGO(..., initialization="distributed"); dpgo_agents_align_async,
dpgo_robust_single_rotation_averaging) against the CPU restatement in tests/dist_init_oracle.py."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import dist_init_oracle as dio  # noqa: E402
from oracle import dpgo_oracle as orc  # noqa: E402

pytestmark = pytest.mark.gpu


def to_meas(edges):
    return orc.Measurements(edges.d, edges.r1, edges.r2, edges.p1, edges.p2, edges.R, edges.t, edges.kappa, edges.tau,
                            edges.weight)


def device_average(RVec, cbar):
    from dpo_b200 import _capi as capi
    lib = capi.load_library()
    m, d = RVec.shape[0], RVec.shape[1]
    R = np.ascontiguousarray(RVec, dtype=np.float64)
    out = np.zeros((d, d))
    flags = np.zeros(m, dtype=np.int32)
    its = C.c_int32(0)
    capi.check(lib.dpgo_robust_single_rotation_averaging(0, d, m, capi.dptr(R), None, cbar, capi.dptr(out),
                                                         capi.iptr(flags), C.byref(its)))
    return out, [int(i) for i in np.flatnonzero(flags)], its.value


@pytest.mark.parametrize("d", [2, 3])
def test_robust_rotation_averaging_kernel_matches_oracle(d):
    """20 seeded fixtures per d (ref tests/testUtils.cpp:90-118 recipe; half of them with outliers just beyond the
    threshold) plus the trivial case: identical inlier sets and GNC iteration counts, R to 1e-12."""
    cases = [dio.rotation_fixture(d, s, near=(s % 2 == 1)) for s in range(20)]
    cases.append((np.array([dio.random_rotation(d, np.random.default_rng(3))] * 4), dio.CBAR))
    for RVec, cbar in cases:
        R, inl, its, _ = dio.robust_single_rotation_averaging(RVec, cbar=cbar)
        Rg, inl_g, its_g = device_average(RVec, cbar)
        assert inl_g == inl and its_g == its
        assert np.abs(Rg - R).max() <= 1e-12


def start(edges, n, k, owner=None, **kw):
    from dpo_b200 import _capi as capi
    from dpo_b200.agent import DistributedPGO
    kw.setdefault("preconditioner", capi.PRECOND_BLOCK_JACOBI)
    return DistributedPGO(edges, n, k, r=5, owner=owner, initialization="distributed", **kw)


def check_against_oracle(run, meas, n, k, owner=None):
    T, Xo, rep = dio.distributed_initialization(meas, n, k, owner=owner)
    assert run.init_report == rep
    X = run.assemble()
    assert np.abs(X - Xo).max() <= 1e-7 * max(1.0, np.abs(Xo).max())
    return T, Xo, rep


@pytest.mark.parametrize("ds,k", [("sphere2500", 5), ("torus3D", 8), ("parking-garage", 4), ("input_INTEL_g2o", 5)])
def test_distributed_start_matches_oracle(ds, k, data_dir):
    from dpo_b200 import posegraph as pg
    edges, n = pg.read_g2o_file(os.path.join(data_dir, ds + ".g2o"))
    meas, _ = orc.read_g2o(os.path.join(data_dir, ds + ".g2o"))
    run = start(edges, n, k)
    _, _, rep = check_against_oracle(run, meas, n, k)
    assert max(r["wave"] for r in rep) >= 1
    assert set(run.init_times) == {"local_chordal_s", "waves_s"}


def test_distributed_start_synthetic_grid_blocks():
    """The lattice of BASELINE config 5 (4 edges per pose) in 8 lattice blocks, at 40 x 40 x 10 so that the oracle's sparse
    direct solves stay fast; the full 100 x 100 x 10 start runs in scripts/bench_configs.py --init distributed."""
    from dpo_b200 import posegraph as pg
    edges, n, _ = pg.synthetic_grid_graph(40, 40, 10, seed=0)
    owner = pg.grid_block_owner(40, 40, 10, 8)
    run = start(edges, n, 8, owner=owner)
    check_against_oracle(run, to_meas(edges), n, 8, owner=owner)


def test_outlier_shared_edges_are_rejected(data_dir):
    """40 % of the loop closures between torus3D agents 0 and 1 replaced by seeded random SE(3) transforms: agent 1 aligns
    to agent 0 on the oracle's inlier set, which holds none of the corrupted candidates."""
    from dpo_b200 import posegraph as pg
    from dpo_b200.agent import contiguous_owner
    edges, n = pg.read_g2o_file(os.path.join(data_dir, "torus3D.g2o"))
    k = 8
    owner = contiguous_owner(n, k)
    a1, a2 = owner[edges.p1], owner[edges.p2]
    between = np.flatnonzero(((a1 == 0) & (a2 == 1)) | ((a1 == 1) & (a2 == 0)))
    rng = np.random.default_rng(11)
    bad = np.sort(rng.choice(between, size=int(round(0.4 * len(between))), replace=False))
    for e in bad:
        edges.R[e] = dio.random_rotation(3, rng)
        edges.t[e] = rng.uniform(-10, 10, size=3)
    meas = to_meas(edges)
    run = start(edges, n, k)
    check_against_oracle(run, meas, n, k)
    # the oracle's candidates of agent 1 against agent 0 and its inlier set
    parts, counts, glob = orc.split_measurements(meas, owner, k)
    T0 = dio.local_initialization(0, int(counts[0]), parts[0][0], parts[0][1])
    T1 = dio.local_initialization(1, int(counts[1]), parts[1][0], parts[1][1])
    YLift = orc.fixed_stiefel_variable(3, 5)
    X0 = YLift @ T0
    cands = dio.alignment_candidates(1, parts[1][2])[0]
    Ts = np.array([dio.candidate_transform(1, e, parts[1][2], T1, X0[:, 4 * j:4 * j + 4], YLift) for j, e in cands])
    _, inl, _, _ = dio.robust_single_rotation_averaging(Ts[:, :3, :3])
    # agent 1's shared edges keep the global edge order
    shared_global = np.flatnonzero((a1 != a2) & ((a1 == 1) | (a2 == 1)))
    corrupted = {q for q, (_, e) in enumerate(cands) if shared_global[e] in set(bad.tolist())}
    assert corrupted and not (set(inl) & corrupted)
    assert run.init_report[1]["neighbor"] == 0 and run.init_report[1]["inliers"] == len(inl)
    _, inl_g, _ = device_average(Ts[:, :3, :3], dio.CBAR)
    assert inl_g == inl


def test_two_runs_bit_identical(data_dir):
    from dpo_b200 import posegraph as pg
    edges, n = pg.read_g2o_file(os.path.join(data_dir, "torus3D.g2o"))
    X = [start(edges, n, 8).assemble() for _ in range(2)]
    assert np.array_equal(X[0], X[1])


@pytest.mark.parametrize("ds,k", [("torus3D", 8), ("sphere2500", 5)])
def test_coloured_rbcd_from_distributed_start(ds, k, data_dir):
    """Coloured RBCD from the distributed start against the oracle's coloured driver from the oracle's distributed start:
    the first 50 rounds at the coloured-parity tolerances of test_gpu_agents, then on to |g| < 0.1, which both must reach
    in the same round at the same 2f (1e-6 relative)."""
    from dpo_b200 import posegraph as pg
    from dpo_b200.agent import DistributedPGO
    edges, n = pg.read_g2o_file(os.path.join(data_dir, ds + ".g2o"))
    meas, _ = orc.read_g2o(os.path.join(data_dir, ds + ".g2o"))
    run = DistributedPGO(edges, n, k, r=5, schedule="coloured", concurrent=False, initialization="distributed")
    T, _, _ = dio.distributed_initialization(meas, n, k)
    drv = orc.MultiRobotDriver(meas, n, k, r=5, schedule="coloured", T_init=T)
    for _ in range(50):
        st = run.step()
        cost, gn = drv.step()
        assert abs(st.cost - cost) <= 1e-8 * abs(cost)
        assert abs(st.gradnorm - gn) <= 1e-7 * gn
    while gn >= 0.1 and drv.round < 1000:
        cost, gn = drv.step()
    while st.gradnorm >= 0.1 and run.round < 1000:
        st = run.step()
    assert gn < 0.1 and st.gradnorm < 0.1
    assert run.round == drv.round
    assert abs(st.cost - cost) <= 1e-6 * abs(cost)


def test_distributed_start_full_size_lattice_known_answer():
    """The 100 x 100 x 10 lattice of BASELINE config 5 (4 edges per pose) in 8 blocks, noise-free: every local chordal
    start is exact in its own frame, so the distributed start is the ground truth in the frame of agent 0's first pose.
    (The oracle comparison of test_distributed_start_synthetic_grid_blocks runs at 40 x 40 x 10: the oracle's sparse direct
    solves take minutes per agent at this size.)"""
    from dpo_b200 import posegraph as pg
    nx, ny, nz, k = 100, 100, 10, 8
    edges, n, Tgt = pg.synthetic_grid_graph(nx, ny, nz, seed=0, rot_sigma=0.0, trans_sigma=0.0)
    owner = pg.grid_block_owner(nx, ny, nz, k)
    run = start(edges, n, k, owner=owner)
    g0 = int(np.flatnonzero(owner == 0)[0])
    H = np.eye(4)
    H[:3] = Tgt[:, 4 * g0:4 * g0 + 4]
    expected = orc.fixed_stiefel_variable(3, 5) @ dio.apply_transform(np.linalg.inv(H), Tgt)
    X = run.assemble()
    assert np.abs(X - expected).max() <= 1e-7 * np.abs(expected).max()
    rep = run.init_report
    assert rep[0]["wave"] == 0 and all(r["wave"] >= 1 and r["inliers"] == r["candidates"] > 0 for r in rep[1:])


def test_align_call_with_an_agent_without_shared_edges(data_dir):
    """An agent with an empty candidate table may share an align call with agents that have candidates: it reports no
    neighbour and keeps its iterate, the others align as usual."""
    from dpo_b200 import _capi as capi
    from dpo_b200 import posegraph as pg
    from dpo_b200.problem import QuadraticProblem
    edges, n = pg.read_g2o_file(os.path.join(data_dir, "torus3D.g2o"))
    run = start(edges, n, 8)
    lone = QuadraticProblem(4, 3, 5)
    lib = lone._lib
    T = np.asfortranarray(np.tile(np.hstack([np.eye(3), np.zeros((3, 1))]), (1, 4)))
    Y = np.asfortranarray(orc.fixed_stiefel_variable(3, 5))
    capi.check(lib.dpgo_agent_set_local_trajectory(lone._h, capi.dptr(T), capi.dptr(Y)))
    capi.check(lib.dpgo_agent_set_align_candidates(lone._h, 0, None, None, None, None, None, None))
    X_lone = lone.download_X()
    X1 = run.agents[1].mProblem.download_X()
    run.exchange(build=False)
    ready = np.zeros(8, dtype=np.int32)
    ready[0] = 1
    hs = (C.c_void_p * 2)(run.agents[1].mProblem._h, lone._h)
    capi.check(lib.dpgo_agents_align_async(hs, 2, C.c_void_p(run.tiles.all.data_ptr()), 8 * run.plan.pmax, capi.iptr(ready), 8,
                                           None))
    info = np.zeros(4, dtype=np.int32)
    capi.check(lib.dpgo_agent_align_result(lone._h, None, capi.iptr(info)))
    assert list(info) == [-1, 0, 0, 0] and np.array_equal(lone.download_X(), X_lone)
    capi.check(lib.dpgo_agent_align_result(run.agents[1].mProblem._h, None, capi.iptr(info)))
    rep = run.init_report[1]
    assert list(info) == [rep["neighbor"], rep["candidates"], rep["inliers"], rep["iterations"]]
    assert np.array_equal(run.agents[1].mProblem.download_X(), X1)     # the same alignment again, bit for bit


def test_cpp_device_runner_matches_python_runner(tmp_path, data_dir):
    """C++ DeviceRBCD with initialization "distributed" (examples/MultiAgentPGO --resident --init distributed) on torus3D /
    8 agents: the same per-agent alignment record as the Python runner, and the same coloured trace from that start.  The
    C++ host's fixedStiefelVariable is a different (equally valid) point of St(3, 5) than the Python one, so the iterates
    agree to rounding, not bitwise; the cost and gradient norm do not depend on the lift."""
    import subprocess
    from dpo_b200 import posegraph as pg
    from dpo_b200.agent import DistributedPGO
    exe = os.path.join(ROOT, "build", "examples", "MultiAgentPGO")
    trace = os.path.join(str(tmp_path), "trace.csv")
    res = subprocess.run([exe, os.path.join(data_dir, "torus3D.g2o"), "--robots", "8", "--iters", "20", "--stop", "0",
                          "--resident", "--schedule", "coloured", "--init", "distributed", "--trace", trace],
                         capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-2000:]
    rec = [[int(v) for v in ln.split()[2:]] for ln in res.stdout.splitlines() if ln.startswith("init ")]
    edges, n = pg.read_g2o_file(os.path.join(data_dir, "torus3D.g2o"))
    run = DistributedPGO(edges, n, 8, r=5, schedule="coloured", initialization="distributed")
    assert rec == [[r["wave"], r["neighbor"], r["candidates"], r["inliers"], r["iterations"]] for r in run.init_report]
    tr = np.loadtxt(trace, delimiter=",").reshape(-1, 4)
    py = np.array([(st.cost, st.gradnorm) for st in (run.step() for _ in range(20))])
    assert np.max(np.abs(tr[:, 2] - py[:, 0]) / py[:, 0]) <= 1e-9
    assert np.max(np.abs(tr[:, 3] - py[:, 1]) / py[:, 1]) <= 1e-7


def test_error_paths(data_dir):
    from dpo_b200 import posegraph as pg
    from dpo_b200.agent import DistributedPGO
    edges, n = pg.read_g2o_file(os.path.join(data_dir, "smallGrid3D.g2o"))
    with pytest.raises(ValueError, match="X_init"):
        DistributedPGO(edges, n, 4, r=5, X_init=np.zeros((5, 4 * n)), initialization="distributed")
    owner = np.minimum(np.arange(n) // (n // 4), 3)
    a1, a2 = owner[edges.p1], owner[edges.p2]
    cut = edges.take(np.flatnonzero(~((a1 != a2) & ((a1 == 3) | (a2 == 3)))))
    with pytest.raises(RuntimeError, match=r"agents \[3\]"):
        start(cut, n, 4)
    g, gn, _ = pg.synthetic_grid_graph(8, 2, 2, edges_per_pose=1.0, seed=0)
    slab_owner = np.array([0, 1, 2, 1])[pg.grid_lattice_coords(8, 2, 2)[:, 0] // 2]
    with pytest.raises(ValueError, match="agent 1"):
        start(g, gn, 3, owner=slab_owner)


def test_two_ranks_bit_equal_to_one_process(tmp_path, data_dir):
    """torus3D / 8 agents over 2 NCCL ranks: the same start, bit for bit, as all agents in one process.  Needs 2 GPUs."""
    import json
    import subprocess
    from dpo_b200 import _capi as capi
    from dpo_b200 import posegraph as pg
    from dpo_b200.agent import DistributedPGO
    cnt = C.c_int(0)
    capi.load_library().dpgo_device_count(C.byref(cnt))
    if cnt.value < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29541", os.path.join(ROOT, "tests", "_dist_init_multirank_worker.py"), "torus3D", "8",
           str(tmp_path)]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-2000:]
    edges, n = pg.read_g2o_file(os.path.join(data_dir, "torus3D.g2o"))
    run = DistributedPGO(edges, n, 8, r=5, schedule="coloured", concurrent=False, initialization="distributed")
    for a in range(8):
        assert np.array_equal(np.load(os.path.join(str(tmp_path), f"X_{a}.npy")), run.agents[a].mProblem.download_X()), a
    with open(os.path.join(str(tmp_path), "report.json")) as fh:
        assert json.load(fh) == run.init_report


def tiny_agent_owner(n):
    """smallGrid3D in 4 agents, agent 1 owning exactly 2 consecutive poses and agent 2 exactly 3 (joined by odometry, and
    sharing odometry edges with agents 0 and 3): their local chordal solves converge before CG's first residual check."""
    owner = np.full(n, 3, dtype=np.int64)
    owner[:60] = 0
    owner[60:62] = 1
    owner[62:65] = 2
    return owner


def test_agents_of_two_and_three_poses(tmp_path, data_dir):
    """The distributed start with agents of 2 and 3 poses, in the Python runner against the oracle and in the C++ device
    runner (examples/MultiAgentPGO --resident --init distributed --partition FILE): the same per-agent records."""
    import subprocess
    from dpo_b200 import posegraph as pg
    path = os.path.join(data_dir, "smallGrid3D.g2o")
    edges, n = pg.read_g2o_file(path)
    meas, _ = orc.read_g2o(path)
    owner = tiny_agent_owner(n)
    parts, counts, _ = orc.split_measurements(meas, owner, 4)
    assert list(counts[1:3]) == [2, 3] and all(len(parts[a][2]) > 0 for a in range(4))
    run = start(edges, n, 4, owner=owner)
    _, _, rep = check_against_oracle(run, meas, n, 4, owner=owner)
    assert all(r["wave"] >= 0 for r in rep)
    part = os.path.join(str(tmp_path), "owner.txt")
    np.savetxt(part, owner, fmt="%d")
    exe = os.path.join(ROOT, "build", "examples", "MultiAgentPGO")
    res = subprocess.run([exe, path, "--robots", "4", "--iters", "1", "--stop", "0", "--resident", "--init", "distributed",
                          "--partition", part], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-2000:]
    rec = [[int(v) for v in ln.split()[2:]] for ln in res.stdout.splitlines() if ln.startswith("init ")]
    assert rec == [[r["wave"], r["neighbor"], r["candidates"], r["inliers"], r["iterations"]] for r in rep]

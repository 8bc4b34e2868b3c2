"""The pose-covariance cases of covariance_cases.py without a GPU: each reaches the regime it is built for (the planner's
host facts, info16), and the host emulation of the device sweep meets the conditioning bound against the
extended-precision reference."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import covariance_cases as cc  # noqa: E402


def _cases(skip=()):
    return [pytest.param(n, d, id=f"{n}-{d}d") for n, d in cc.CASES if n not in skip]


SEL_T, SEL_K = 64, 32          # dpgo_covariance.cu: output tile and inner chunk of the sweep's products

# info16 facts each case must show: (levels, macro nodes, largest own block, largest boundary) per d; None = not fixed
TARGETS = {
    "pair": {2: (1, 1, 6, 0), 3: (1, 1, 12, 0)},
    "pair_multi": {2: (1, 1, 6, 0), 3: (1, 1, 12, 0)},
    "triangle": {2: (1, 1, 9, 0), 3: (1, 1, 18, 0)},
    "hub2100_anchor_hub": {2: (2, 257, None, 0), 3: (2, 513, None, 0)},
    "hub2100_anchor_leaf": {2: (2, 257, None, 3), 3: (2, 513, None, 6)},
    "star191_chain_hub": {2: (1, 1, 576, 0), 3: (2, None, None, None)},
    "star191_chain_leaf": {2: (1, 1, 576, 0), 3: (2, None, None, None)},
    "clique60": {2: (1, 1, 180, 0), 3: (1, 1, 360, 0)},
    "clique200": {2: (1, 1, 600, 0), 3: (1, 1, 1200, 0)},
    "lattice30x30": {2: (None, None, None, 84), 3: (None, None, None, 168)},
}


@pytest.mark.parametrize("name,d", _cases(skip=("single",)))
def test_case_reaches_its_target(name, d):
    case = cc.make_case(name, d)
    _, _, info = cc.emulate(case)
    assert info[2] == case.n * case.b // 3
    want = TARGETS.get(name, {}).get(d)
    if want is not None:
        got = (info[0], info[1], info[5], info[6])
        assert all(w is None or g == w for g, w in zip(got, want)), (got, want)
    if name.startswith("path5000"):
        assert info[0] == (2 if d == 2 else 3) and info[1] <= 1089 and info[6] > 0
    if name in ("lattice30x30", "graded", "path2000_pairs"):
        assert info[6] > SEL_T and info[6] % SEL_K != 0                     # boundary tiles past SEL_T, a partial SEL_K chunk
    if name == "path2000_pairs":
        ij = {tuple(p) for p in case.pairs.tolist()}
        assert any((j, i) in ij for i, j in ij if i != j)
        assert len(ij) < len(case.pairs) and any(i == j for i, j in ij)
        assert any(case.anchor in p for p in ij)
    if name in ("pair_multi", "multi_edges"):
        pe = list(zip(case.edges.p1.tolist(), case.edges.p2.tolist()))
        assert len(set(pe)) < len(pe)                                        # a duplicated edge
        assert any((j, i) in set(pe) for i, j in pe)                          # both directions
    if name == "path600k":
        assert info[13] > cc.MAX_GRID_YZ
    else:
        assert 1 <= info[13] <= info[1]


@pytest.mark.parametrize("name,d", _cases(skip=("single", "path600k")))
def test_host_emulation_meets_the_bound(name, d):
    case = cc.make_case(name, d)
    ref = cc.reference(name, d)
    cov, pc, _ = cc.emulate(case)
    poses = ref.sample()
    pp = [(int(p), int(p)) for p in poses]
    r = cc.worst_ratio(ref, cov[poses], ref.blocks(pp), pp)
    assert r <= cc.C_BOUND, (case.id, r, ref.kappa)
    if len(case.pairs):
        r = cc.worst_ratio(ref, pc, ref.blocks(case.pairs), case.pairs)
        assert r <= cc.C_BOUND, (case.id, r, ref.kappa)
    for p, S in case.closed.items():
        r = cc.worst_ratio(ref, cov[[p]], [S], [(p, p)])
        assert r <= cc.C_BOUND, (case.id, p, r)
    assert np.all(cov[case.anchor] == 0)


@pytest.mark.parametrize("d", [2, 3])
def test_graded_case_is_ill_conditioned_but_not_singular(d):
    """the diagonal of H spans more than 1e12 (so its plain condition number is at least that), while the scaled
    condition number keeps the bound well below the blocks' own size"""
    ref = cc.reference("graded", d)
    assert ref.h.max() / ref.h.min() > 1e12, ref.h.max() / ref.h.min()
    assert cc.C_BOUND * cc.U * ref.kappa < 1e-3, ref.kappa


@pytest.mark.parametrize("d", [2, 3])
def test_single_pose_returns_zeros_without_a_device(d):
    """n = 1 (the anchor alone) returns before any device call, so it succeeds on a machine without a GPU"""
    from dpo_b200 import _capi as capi
    case = cc.make_case("single", d)
    code, cov, pc, info = cc.call_device(case, device=0)
    assert code == 0, capi.last_error()
    assert np.array_equal(cov, np.zeros_like(cov)) and np.array_equal(pc, np.zeros_like(pc))
    assert info == [0] * 16


def test_gauss_jordan_arithmetic_misses_the_bound_on_the_graded_3d_lattice():
    """Why the device misses the bound on the graded 3D lattice (test_gpu_covariance_cases.py marks it as an expected
    failure).  The device inverts every front by blocked Gauss-Jordan sweeps.  The same arithmetic on the whole anchored
    information, in fp64 on the host, misses the bound by far at the tiny-kappa pose and its neighbours, while a Cholesky
    inverse of the very same fp64 matrix meets it with room to spare.  So the loss is in Gauss-Jordan elimination itself,
    not in a kernel defect.  A power-of-two Jacobi scaling cannot recover it: every operation of the sweep scales exactly,
    so the sweep of the scaled matrix, scaled back, is bitwise the sweep of the matrix."""
    import scipy.linalg as sl
    ref = cc.reference("graded", 3)
    case, b = ref.case, ref.case.b
    H = ref.Hf.toarray()
    G = cc.gauss_jordan_inverse(H)
    Ch = sl.cho_solve(sl.cho_factor(H, lower=True), np.eye(len(H)))
    pp = [(p, p) for p in case.watch]
    want = ref.blocks(pp)

    def blocks(X):
        f = [(p - (p > case.anchor)) * b for p in case.watch]               # free index of each pose's first scalar
        return [X[i:i + b, i:i + b] for i in f]

    gj, ch = cc.worst_ratio(ref, blocks(G), want, pp), cc.worst_ratio(ref, blocks(Ch), want, pp)
    assert gj > cc.C_BOUND and ch < 1.0, (gj, ch)
    s = 2.0 ** np.round(-0.5 * np.log2(np.diag(H)))
    assert np.array_equal(cc.gauss_jordan_inverse(H * s[:, None] * s[None, :]) * s[:, None] * s[None, :], G)

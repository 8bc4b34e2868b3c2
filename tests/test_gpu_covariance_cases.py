"""Pose covariances on the GPU (dpgo_pose_covariances) on the graphs of covariance_cases.py: against the
extended-precision reference within the conditioning bound, against closed forms, exact properties (repeatability,
anchor zeros, symmetry, pair transposes, power-of-two scaling), the host emulation, and a stage of more than 65535 macro
nodes."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import covariance_cases as cc  # noqa: E402

pytestmark = pytest.mark.gpu

# The device misses the bound on the 3D graded lattice, at pose 464 (next to the pose whose rotation only a tiny kappa
# holds): 755 u k^ ||H^^-1|| / sqrt(h h) against the reference where the host emulation's Cholesky fronts stay at 0.15.
# test_covariance_cases_cpu.py::test_gauss_jordan_arithmetic_misses_the_bound_on_the_graded_3d_lattice shows the cause:
# the device's blocked Gauss-Jordan arithmetic, emulated in fp64 on this matrix, misses the bound by as much, where a
# Cholesky inverse of the same matrix meets it.  Kept as a strict expected failure so that the finding stays visible and
# a Cholesky-based front inverse on the device shows up as an unexpected pass.
GRADED_3D = pytest.mark.xfail(strict=True, reason="device Gauss-Jordan fronts exceed the bound on the graded 3D lattice")
ACCURACY = [pytest.param(n, d, id=f"{n}-{d}d", marks=GRADED_3D if (n, d) == ("graded", 3) else ())
            for n, d in cc.CASES if n not in ("single", "path600k")]
CASES = [pytest.param(n, d, id=f"{n}-{d}d") for n, d in cc.CASES if n not in ("single", "path600k")]
_runs = {}


def run(name, d):
    """the case and one device call, once per process"""
    if (name, d) not in _runs:
        from dpo_b200 import _capi as capi
        case = cc.make_case(name, d)
        code, cov, pc, info = cc.call_device(case)
        assert code == 0, (case.id, code, capi.last_error())
        _runs[(name, d)] = (case, cov, pc, info)
    return _runs[(name, d)]


def _pose_pairs(poses):
    return [(int(p), int(p)) for p in poses]


@pytest.mark.parametrize("name,d", ACCURACY)
def test_blocks_meet_the_bound_against_the_reference(name, d):
    case, cov, pc, _ = run(name, d)
    ref = cc.reference(name, d)
    pp = _pose_pairs(ref.sample())
    worst = cc.worst_ratio(ref, cov[[p for p, _ in pp]], ref.blocks(pp), pp)
    assert worst <= cc.C_BOUND, (case.id, worst, ref.kappa)
    if len(case.pairs):
        r = cc.worst_ratio(ref, pc, ref.blocks(case.pairs), case.pairs)
        assert r <= cc.C_BOUND, (case.id, r, ref.kappa)
        worst = max(worst, r)
    if case.closed:                       # every closed-form block, within C u k^ of its own scale
        ps = sorted(case.closed)
        r = cc.worst_ratio(ref, cov[ps], [case.closed[p] for p in ps], _pose_pairs(ps))
        assert r <= cc.C_BOUND, (case.id, r)
        worst = max(worst, r)
    print(f"\n{case.id}: k^ = {ref.kappa:.3g}, largest error / bound = {worst / cc.C_BOUND:.3g}")


@pytest.mark.parametrize("name,d", CASES)
def test_exact_properties(name, d):
    case, cov, pc, _ = run(name, d)
    _, cov2, pc2, _ = cc.call_device(case)
    assert np.array_equal(cov, cov2) and np.array_equal(pc, pc2)                       # two calls are bitwise equal
    a = case.anchor
    assert np.all(cov[a] == 0)
    for p in range(case.n):
        if p != a:
            assert np.array_equal(cov[p], cov[p].T), p
    free = [p for p in range(case.n) if p != a]
    assert np.all(np.linalg.eigvalsh(cov[free])[:, 0] > 0)
    where = {}
    for k, (i, j) in enumerate(case.pairs.tolist()):
        if a in (i, j):
            assert np.all(pc[k] == 0), (i, j)
        if i == j:
            assert np.array_equal(pc[k], cov[i]), (i, j)
        if (i, j) in where:
            assert np.array_equal(pc[k], pc[where[(i, j)]]), (i, j)                   # duplicated pair
        if (j, i) in where:
            assert np.array_equal(pc[k], pc[where[(j, i)]].T), (i, j)                 # both orders
        where.setdefault((i, j), k)


@pytest.mark.parametrize("name,d", CASES)
def test_power_of_two_scaling_is_exact(name, d):
    """Every operation of the assembly, the Gauss-Jordan sweeps and the selected inversion scales exactly by a power of
    two, so kappa, tau times 2^10 gives Sigma times 2^-10 and weights times 2^-10 give Sigma times 2^10, bit for bit."""
    case, cov, pc, _ = run(name, d)
    e = case.edges
    up = e.take(np.arange(len(e)))
    up.kappa, up.tau = e.kappa * 2.0 ** 10, e.tau * 2.0 ** 10
    code, c1, p1, _ = cc.call_device(case, edges=up)
    assert code == 0 and np.array_equal(c1, cov * 2.0 ** -10) and np.array_equal(p1, pc * 2.0 ** -10)
    down = e.take(np.arange(len(e)))
    down.weight = e.weight * 2.0 ** -10
    code, c2, p2, _ = cc.call_device(case, edges=down)
    assert code == 0 and np.array_equal(c2, cov * 2.0 ** 10) and np.array_equal(p2, pc * 2.0 ** 10)


@pytest.mark.parametrize("name,d", ACCURACY)
def test_device_meets_the_bound_against_the_host_emulation(name, d):
    """the device factors by Gauss-Jordan, the host emulation by build_numeric: both within the bound of each other"""
    case, cov, pc, info = run(name, d)
    ref = cc.reference(name, d)
    hc, hp, hinfo = cc.emulate(case)
    assert hinfo[:10] == info[:10] and hinfo[13] == info[13]
    assert np.array_equal(hc[case.anchor], cov[case.anchor])
    assert cc.worst_ratio(ref, cov, hc, _pose_pairs(range(case.n))) <= cc.C_BOUND
    if len(case.pairs):
        assert cc.worst_ratio(ref, pc, hp, case.pairs) <= cc.C_BOUND


def test_a_stage_of_more_than_65535_macro_nodes():
    """A 600000-pose path: the dissection's deepest stage has more macro nodes than one launch's blockIdx.y / z can
    index, so the factorisation and the sweep run it in slices.  The call succeeds and its sampled blocks meet the bound
    (16 poses: each is three column solves over 1.8 million unknowns, refined in long double)."""
    from dpo_b200 import _capi as capi
    case = cc.make_case("path600k", 2)
    code, cov, _, info = cc.call_device(case)
    assert code == 0, capi.last_error()
    assert info[13] > cc.MAX_GRID_YZ, info
    ref = cc.reference("path600k", 2)
    pp = _pose_pairs(ref.sample(16))
    r = cc.worst_ratio(ref, cov[[p for p, _ in pp]], ref.blocks(pp), pp)
    assert r <= cc.C_BOUND, (r, ref.kappa)
    assert np.all(cov[case.anchor] == 0)
    print(f"\npath600k-2d: k^ = {ref.kappa:.3g}, largest error / bound = {r / cc.C_BOUND:.3g}, stage of {info[13]} macro nodes")

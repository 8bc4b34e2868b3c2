"""CPU checks of the RTR cases of rtr_cases.py: every case reaches the trust-region branch it is built for, judged from
the oracle's decision trace, with every decision on its path clear of its threshold; a wrong variant of the case's branch
changes what the GPU test compares; and the oracle's give-up count and its exactly stationary start agree with the
kernel's documented behaviour."""
import numpy as np
import pytest

import rtr_cases as rc

PARAMS = [(d, r, p) for d in (2, 3) for r in rc.RANKS[d] for p in rc.PRECONDS]


@pytest.mark.parametrize("d,r,precond", PARAMS)
@pytest.mark.parametrize("name", rc.CASE_NAMES)
def test_case_reaches_its_branch(name, d, r, precond):
    c = rc.case(name, d, r, precond)
    assert rc.REACHES[name][1](c), (c.target, c.attempts())
    what, worst = min(rc.margins(c.trace), key=lambda m: m[1])
    assert worst >= rc.margin_floor(precond), (c.target, what, worst)


@pytest.mark.parametrize("d,r,precond", PARAMS)
@pytest.mark.parametrize("name", sorted(rc.MUTATIONS))
def test_mutations_change_what_the_gpu_compares(name, d, r, precond):
    c = rc.case(name, d, r, precond)
    for m in c.mutations:
        Xm, res, _ = rc.run(c.Q, c.G, c.X, d, r, precond, c.tol, c.iters, c.inner, c.radius, m)
        assert rc.differs(c, Xm, res, rc.tolerances(precond)), (name, m)


def test_every_mutation_has_a_case():
    assert {m for ms in rc.MUTATIONS.values() for m in ms} == {"no_cap", "shrink_half", "accept_positive", "giveup_11",
                                                               "stale_z0", "wrong_root"}
    assert set(rc.MUTATIONS) <= set(rc.CASE_NAMES)


@pytest.mark.parametrize("precond", rc.PRECONDS)
def test_rejections_count_the_attempt_before_the_giveup(precond):
    c = rc.case("giveup", 3, 5, precond)
    assert c.result.outer_iterations == 12 and c.result.rejections == 12
    assert all(a[2] < 1e-20 for a in c.attempts())
    assert np.array_equal(c.X_out, c.X) and c.result.fOpt == c.result.fInit


@pytest.mark.parametrize("precond", rc.PRECONDS)
@pytest.mark.parametrize("d", [2, 3])
def test_stationary_start_returns_its_input(d, precond):
    """g = 0 exactly and tolerance 0: no ZeroDivisionError; every attempt is rejected (tau = 0, model decrease 0) and
    the step gives up with the input, bit for bit"""
    c = rc.case("stationary", d, rc.RANKS[d][0], precond)
    res = c.result
    assert res.gradNormInit == 0.0 and res.fInit == 0.0
    assert (res.tcg_status, res.tcg_iterations, res.outer_iterations, res.rejections) == (rc.NEGCURV, 12, 12, 12)
    assert np.array_equal(c.X_out, c.X)
    assert res.relativeChange == 0.0 and res.fOpt == res.fInit and res.gradNormOpt == res.gradNormInit


def test_batch_agents_cover_giveup_reject_accept():
    for d, r in rc.BATCH_DR:
        agents = rc.batch_agents(d, r)
        assert [a.result.rejections for a in agents] == [12, 1, 0]
        assert len({(a.tol, a.iters, a.inner, a.radius) for a in agents}) == 1
        assert all(a.G is None or not a.G.any() for a in agents)
        for a in agents:
            assert rc.min_margin(a.trace) >= rc.margin_floor("exact")

"""CPU checks of the multi-agent cases of agent_cases.py: every case reaches the branch it is built for, from host facts
and the kernels' constants alone, and the references and host rules have the power to tell the kernel from a subtly
wrong one."""
import numpy as np
import pytest

import agent_cases as ac
import dist_init_oracle as dio
import structure_cases as sc
from oracle import dpgo_oracle as orc


def test_status_sizes_reach_the_second_trip():
    ctas = [ac.status_ctas(n) for n in ac.SIZES]
    assert 1 in ac.SIZES and any(n % 32 == 0 for n in ac.SIZES)
    assert max(ctas) > 32 and sum(c > 32 for c in ctas) >= 5        # the lane-strided final sum takes a 2nd / 3rd trip
    assert max(ctas) > 64
    assert ac.status_ctas(1024) == 32 and ac.status_ctas(1025) == 33  # both sides of the first extra trip


def test_small_agent_launch_has_many_jobs():
    s = ac.small_sizes()
    assert len(s) >= 100 and min(s) == 1 and max(s) <= 40 and len(set(s)) >= 30
    assert len(s) > 16                                                # the job search runs deeper than 4 levels
    assert sum(ac.status_ctas(n) for n in s) > len(s)                 # agents of 2 CTAs among them


def test_table_eviction_needs_more_lists_than_the_cache():
    assert 40 > ac.STATUS_TABLES_MAX


def test_accel_sizes_reach_the_second_trip_and_late_ctas():
    assert ac.accel_ctas(4097) == 33 and ac.accel_ctas(5000) == 40
    assert 1 in ac.ACCEL_SIZES
    for n in ac.ACCEL_SIZES:
        p = ac.public_poses(n, "spread")
        cta = set((p // ac.ACCEL_THREADS).tolist())
        assert 0 in cta and ac.accel_ctas(n) - 1 in cta               # first and last CTA
        if ac.accel_ctas(n) > 2:
            assert len(cta) == ac.accel_ctas(n)                        # every CTA, the middle ones included
        assert len(set(p.tolist())) == len(p)
    a = ac.public_poses(4097, "all")
    assert sorted(a.tolist()) == list(range(4097)) and (a != np.arange(4097)).any()
    assert len(ac.public_poses(33, "none")) == 0


@pytest.mark.parametrize("d", [2, 3])
def test_shared_edges_hub(d):
    s = ac.SharedEdges(d, 5, 300)
    hub = s.local == s.hub
    assert (s.out[hub] == 1).sum() >= 300 and (s.out[hub] == 0).sum() >= 300
    rows = np.concatenate([s.local[:, None], s.out[:, None], s.slot[:, None], s.T.reshape(len(s.T), -1), s.om], axis=1)
    assert len(np.unique(rows, axis=0)) < len(rows)                    # exact duplicates
    assert (s.out[:-1] != s.out[1:]).sum() > 100                       # directions interleaved in the input
    assert {0, 299} <= set(s.local.tolist())
    assert (np.abs(s.om[:, :d] - s.om[:, d:]) > 1e-3).all()           # om[q] != om[c]: weighting inside the loop differs


@pytest.mark.parametrize("d", [2, 3])
def test_G_reference_has_power(d):
    """the float64 formula passes the bound; weighting each incoming term by om[q] inside the sum does not"""
    s = ac.SharedEdges(d, 3, 300)
    G, bound = s.G_ref()
    g = s.gathered
    dh = d + 1
    G64 = np.zeros((3, 300, dh))
    Gm = np.zeros((3, 300, dh))
    for k in range(len(s.local)):
        Xn, T, om = g[s.slot[k]], s.T[k], s.om[k]
        if s.out[k]:
            L = Lm = (Xn * om[None, :]) @ T.T
        else:
            L = (Xn @ T) * om[None, :]
            Lm = (Xn * om[None, :]) @ T
        G64[:, s.local[k]] -= L
        Gm[:, s.local[k]] -= Lm
    assert (abs(sc.ld(G64.reshape(3, -1)) - G) <= bound).all()
    assert not (abs(sc.ld(Gm.reshape(3, -1)) - G) <= bound).all()


def test_selection_inputs_reach_their_branches():
    ks = ac.SELECT_KS
    assert max(ks) == ac.SELECT_MAX_AGENTS and any(k > 32 and k % 32 for k in ks)
    assert {ac.graph_kind_for(k) for k in ks} == set(ac.GRAPH_KINDS)
    rec = ac.selection_records(100, 140)
    g = rec[:, :, 2]
    assert rec.shape[0] > 128                                          # the log is read back across its 64 -> 128 doubling
    assert np.isnan(g).any() and np.isposinf(g).any()
    assert ((g == 0) & np.signbit(g)).any() and ((g == 0) & ~np.signbit(g)).any()
    assert ((g > 0) & (g < 2.2250738585072014e-308)).any()
    row = g[0][~np.isnan(g[0])]
    assert len(np.unique(row)) < len(row)                              # exact ties within a round
    for k in ks:
        ptr, adj = ac.agent_graph(k, ac.graph_kind_for(k))
        assert len(ptr) == k + 1 and (adj != np.repeat(np.arange(k), np.diff(ptr))).all()


@pytest.mark.parametrize("k", [31, 33, 100, 1023])
def test_selection_records_tell_the_rule_from_its_mutants(k):
    """over the rounds a GPU test runs, the records give a different mask without the tie rule than with it; an agent
    with a NaN norm and no neighbour is still taken"""
    ptr, adj = ac.agent_graph(k, ac.graph_kind_for(k))
    rec = ac.selection_records(k, 10)
    full = [ac.host_select(rec[i, :, 2], ptr, adj) for i in range(10)]
    no_tie = [ac.host_select(rec[i, :, 2], ptr, adj, tie_rule=False) for i in range(10)]
    assert any((a != b).any() for a, b in zip(full, no_tie))
    for i in range(10):                                                # a NaN never ranks ahead of a number
        g = rec[i, :, 2]
        for a in np.flatnonzero(np.isnan(g)):
            nb = adj[ptr[a]:ptr[a + 1]]
            if not len(nb):
                assert full[i][a] == 1


def test_host_select_keeps_inf_and_signed_zero():
    ptr, adj = ac.agent_graph(3, "path")
    assert ac.host_select(np.array([1e308, np.inf, 0.0]), ptr, adj).tolist() == [0, 1, 0]
    assert ac.host_select(np.array([-0.0, 0.0, np.nan]), ptr, adj).tolist() == [1, 0, 1]     # -0 == +0: lower id first
    assert ac.host_select(np.array([np.nan, 0.0, 0.0]), ptr, adj).tolist() == [0, 1, 0]


@pytest.mark.parametrize("d", [2, 3])
def test_rotation_inputs(d):
    for m in ac.ROT_MS:
        R = ac.rotation_inputs(d, m)
        assert R.shape == (m, d, d)
        assert np.abs(np.einsum("mij,mkj->mik", R, R) - np.eye(d)).max() <= 1e-14
    assert max(ac.ROT_MS) > 4 * ac.ALIGN_THREADS and {255, 256, 257} <= set(ac.ROT_MS)
    assert ac.gnc_skipped(ac.rotation_inputs(d, 1), dio.CBAR) and ac.gnc_skipped(ac.rotation_inputs(d, 2), dio.CBAR)
    assert ac.gnc_skipped(ac.rotation_inputs(d, 1000, all_inlier=True), dio.CBAR)
    assert not ac.gnc_skipped(ac.rotation_inputs(d, 1000), dio.CBAR)


def test_status_reference_has_power():
    a = ac.Agent(3, 4, 1025, 0)
    rec = np.zeros(5)
    XQ = (a.Q @ a.X.T).T
    rec[0] = np.sum(XQ * a.X)
    rec[1] = np.sum(a.X * a.G)
    P = orc.tangent_project(a.X, XQ + a.G, 3)
    rec[2] = np.sum(P * P)
    ac.check_status(rec, a, a.X, "float64 stand-in")
    # the last CTA's 32 rows left out of every field
    Xc = a.X.copy()
    Xc[:, 1024 * 4:] = 0.0
    XQc = (a.Q @ Xc.T).T
    bad = rec.copy()
    bad[0] = np.sum(XQc * Xc)
    with pytest.raises(AssertionError):
        ac.check_status(bad, a, a.X, "last CTA dropped")
    assert sc.U == ac.U


def test_relative_change_reference_has_power():
    rng = np.random.default_rng(0)
    X, XP = rng.standard_normal((5, 4 * 4097)), rng.standard_normal((5, 4 * 4097))
    ref, rel = ac.relative_change_ref(X, XP, 4097)
    got = np.sqrt(np.sum((X - XP) ** 2) / 4097)
    assert abs(got - float(ref)) <= rel * float(ref)
    assert abs(np.sqrt(np.sum((X - XP) ** 2) / ac.accel_ctas(4097)) - float(ref)) > rel * float(ref)
    part = np.sqrt(np.sum((X[:, :4 * 4096] - XP[:, :4 * 4096]) ** 2) / 4097)      # the 33rd CTA's partial dropped
    assert abs(part - float(ref)) > rel * float(ref)

"""The batched multi-agent kernels on the cases of agent_cases.py, driven through the C ABI on QuadraticProblem handles:
team status (k_agents_status), momentum begin and finish (k_accel_agents, k_accel_finish), greedy independent-set
selection (k_select_independent), the G build from shared edges (k_build_G) and the robust rotation averaging of the
frame alignment (k_robust_rotation_average), against long-double references and the host rules; and the refusal of a
handle listed twice in one batched call."""
import ctypes as C

import numpy as np
import pytest

import agent_cases as ac
import dist_init_oracle as dio
import structure_cases as sc
from oracle import dpgo_oracle as orc

pytestmark = pytest.mark.gpu

DR = [(d, r) for d in (2, 3) for r in sc.RANKS[d]]
ERR_INVALID_ARG = 1


def capi():
    from dpo_b200 import _capi
    return _capi


def lib():
    return capi().load_library()


def handle(a: ac.Agent):
    import dpo_b200 as dp
    gp = dp.QuadraticProblem(a.n, a.d, a.r, preconditioners=(dp.PRECOND_BLOCK_JACOBI,))
    gp.setQ(a.Q)
    gp.setG(a.G)
    gp.upload_X(a.X)
    return gp


def handles(gps):
    return (C.c_void_p * len(gps))(*[g._h for g in gps])


def ptrs(ts):
    return (C.c_void_p * len(ts))(*[C.c_void_p(t.data_ptr()) if t is not None else None for t in ts])


def params():
    import dpo_b200 as dp
    prm = capi().OptParams()
    lib().dpgo_opt_params_default(C.byref(prm))
    prm.precond = dp.PRECOND_BLOCK_JACOBI
    return prm


def nan_tensor(count):
    import torch
    return torch.full((max(count, 1),), float("nan"), dtype=torch.float64, device="cuda")


def status(gps, slots, nslots):
    """one dpgo_agents_status_async launch into a NaN-filled buffer of nslots records"""
    import torch
    buf = nan_tensor(nslots * ac.STATUS_DOUBLES)
    sl = np.ascontiguousarray(slots, dtype=np.int32)
    torch.cuda.synchronize()
    capi().check(lib().dpgo_agents_status_async(handles(gps), len(gps), capi().iptr(sl), C.c_void_p(buf.data_ptr()), None))
    for g in gps[:1]:
        g.sync()
    torch.cuda.synchronize()
    return buf.cpu().numpy().reshape(nslots, ac.STATUS_DOUBLES)


def G_reader(gp):
    """reads G through its device address, fetched once: dpgo_problem_device_G marks G as written by the caller, so the
    next G build would clear it first"""
    ptr = gp.device_G_ptr()
    return lambda: read_G(gp, ptr)


def read_G(gp, ptr):
    out = np.empty(gp.r * gp.N)
    gp.sync()
    capi().check(lib().dpgo_copy_to_host_async(gp.device, C.c_void_p(out.ctypes.data), C.c_void_p(ptr), out.nbytes, None))
    capi().check(lib().dpgo_stream_synchronize(gp.device, None))
    return out.reshape(gp.r, gp.N, order="F")


def tile(M, p, d):
    return M[:, p * (d + 1):(p + 1) * (d + 1)]


def send_tile(buf, s, r, d):
    """slot s of a send buffer: one r x (d+1) tile, column-major"""
    ts = r * (d + 1)
    return buf[s * ts:(s + 1) * ts].reshape(d + 1, r).T


# ---------------------------------------------------------------------------------------------------------------------
# team status
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d,r", DR)
def test_status_records(d, r):
    """Agents of 1 .. 5000 poses in one launch (up to 157 CTAs per agent: the final sum's 2nd to 5th trip) and 122 agents
    in another: fields 0-2 within the long-double bounds, 3-4 the agent's last optimising call, each record at its slot
    (permuted), bitwise the same alone, inside the large launch, on a repeated call and after the job-table cache of the
    first agent was cycled by 40 other lists."""
    import dpo_b200 as dp
    big = [ac.Agent(d, r, n, 0) for n in ac.SIZES]
    small = [ac.Agent(d, r, n, 1 + i) for i, n in enumerate(ac.small_sizes())]
    hb, hs = [handle(a) for a in big], [handle(a) for a in small]
    opt_rec = {}
    for i in (3, 5):                                         # an optimising call: fields 3-4 not those of a new handle
        opt = dp.QuadraticOptimizer(hb[i])
        opt.setPreconditioner(dp.PRECOND_BLOCK_JACOBI)
        opt.optimize_resident_async()
        opt_rec[i] = (opt.fetch_result().relative_change, 1.0)
    Xb = [g.download_X() for g in hb]
    rng = np.random.default_rng([d, r])
    perm = rng.permutation(len(big) + 3)[:len(big)]          # slots permuted, with gaps
    rec = status(hb, perm, len(big) + 3)
    assert np.isnan(rec[np.setdiff1d(np.arange(len(big) + 3), perm)]).all()
    for i, a in enumerate(big):
        ac.check_status(rec[perm[i]], a, Xb[i], f"n={a.n}")
        assert tuple(rec[perm[i], 3:]) == opt_rec.get(i, (0.0, 0.0)), a.n
    assert np.array_equal(status(hb, perm, len(big) + 3), rec, equal_nan=True)   # ticket reset by the last CTA
    for i in range(len(big)):
        assert np.array_equal(status([hb[i]], [0], 1)[0], rec[perm[i]]), big[i].n
    # 122 agents: the small ones with two large ones among them
    mixed = hs[:50] + [hb[5]] + hs[50:] + [hb[9]]
    mperm = rng.permutation(len(mixed))
    mrec = status(mixed, mperm, len(mixed))
    assert np.array_equal(mrec[mperm[50]], rec[perm[5]]) and np.array_equal(mrec[mperm[-1]], rec[perm[9]])
    for j, a in enumerate(small):
        slot = mperm[j if j < 50 else j + 1]
        ac.check_status(mrec[slot], a, a.X, f"small agent {j}, n={a.n}")
        assert tuple(mrec[slot, 3:]) == (0.0, 0.0)
    # 40 more lists with the same first agent evict the first list's job table
    for j in range(40):
        status([hb[0], hs[j]], [1, 0], 2)
    assert np.array_equal(status(hb, perm, len(big) + 3), rec, equal_nan=True)


# ---------------------------------------------------------------------------------------------------------------------
# momentum begin and finish
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("restart", [False, True], ids=["plain", "restart"])
@pytest.mark.parametrize("d,r", DR)
def test_accel_begin_and_finish(d, r, restart):
    """Two begin launches of five agents (1 .. 5000 poses), the second mixed active / idle and, with restart_interval 3,
    a restart round.  X, Y and the momentum record against the references (V is the iterate at dpgo_agent_accel_init,
    untouched by the first round's active begin), public tiles in their slots and nothing past them; then the active
    agents' round, whose status record holds sqrt(|X - XPrev|^2 / n) within its bound and one optimising call."""
    import torch
    L, cp = lib(), capi()
    N_mom, ri = 5.0, (3 if restart else 30)
    agents = [ac.Agent(d, r, n, 7) for n in ac.ACCEL_SIZES]
    kinds = ["all", "none", "all", "all", "spread"]
    active2 = np.array([0, 1, 0, 1, 1], dtype=np.int32)
    gps = [handle(a) for a in agents]
    pubs = [ac.public_poses(a.n, k, seed=d * 10 + r) for a, k in zip(agents, kinds)]
    ts = r * (d + 1)
    for g, p in zip(gps, pubs):
        cp.check(L.dpgo_agent_set_public_poses(g._h, len(p), cp.iptr(p) if len(p) else None))
        cp.check(L.dpgo_agent_accel_init(g._h))
    sx = [nan_tensor((len(p) + 2) * ts) for p in pubs]       # two tiles past the last slot must stay NaN
    sy = [nan_tensor((len(p) + 2) * ts) for p in pubs]
    hs = handles(gps)

    def begin(flags):
        torch.cuda.synchronize()
        cp.check(L.dpgo_agents_accel_begin_async(hs, len(gps), cp.iptr(np.ascontiguousarray(flags, dtype=np.int32)), N_mom,
                                                 ri, ptrs(sx), ptrs(sy), None))
        gps[0].sync()
        torch.cuda.synchronize()

    begin(np.ones(5, dtype=np.int32))                        # round 1: every agent active, so V stays X0
    rng = np.random.default_rng([d, r, 2])
    X2 = [orc.manifold_project(rng.standard_normal((r, a.case.N)), d) for a in agents]
    for g, X in zip(gps, X2):
        g.upload_X(X)
    for t in sx + sy:
        t.fill_(float("nan"))
    begin(active2)
    g1 = ac.momentum_gamma(0.0, N_mom)
    g2 = ac.momentum_gamma(g1, N_mom)
    a2 = ac.momentum_alpha(g2, N_mom)
    for i, (a, g) in enumerate(zip(agents, gps)):
        what = f"n={a.n} active={active2[i]}"
        st = np.zeros(3)
        cp.check(L.dpgo_agent_accel_state(g._h, cp.dptr(st)))
        assert tuple(st) == ((0.0, 0.0, 2.0) if restart else (g2, a2, 2.0)), what
        Xa = g.download_X()
        bx, by = sx[i].cpu().numpy(), sy[i].cpu().numpy()
        p = pubs[i]
        assert np.isnan(bx[len(p) * ts:]).all() and np.isnan(by[len(p) * ts:]).all(), what
        Yg = np.full_like(Xa, np.nan)
        for s, pose in enumerate(p):
            assert np.array_equal(send_tile(bx, s, r, d), tile(Xa, pose, d)), (what, s)
            Yg[:, pose * (d + 1):(pose + 1) * (d + 1)] = send_tile(by, s, r, d)
        idle = not active2[i]
        if idle and restart:                                 # X = XPrev, V = Y = X
            assert np.array_equal(Xa, X2[i]), what
            for s, pose in enumerate(p):
                assert np.array_equal(send_tile(by, s, r, d), tile(X2[i], pose, d)), (what, s)
            continue
        if idle:                                             # X = Y
            for pose in p:
                assert np.array_equal(tile(Xa, pose, d), tile(Yg, pose, d)), (what, pose)
        else:
            assert np.array_equal(Xa, X2[i]), what
        if len(p):
            M, Mm = ac.momentum_M(X2[i], a.X, a2)
            ac.check_polar_step(Yg, M, Mm, d, np.sort(p), what)
    # the active agents' part of the round, then their status records
    act = [gps[i] for i in np.flatnonzero(active2)]
    prm = params()
    torch.cuda.synchronize()
    cp.check(L.dpgo_agents_accel_round_async(handles(act), len(act), C.byref(prm), None, None, 0, None))
    for g in act:
        g.sync()
    rec = status(gps, np.arange(5), 5)
    for i, (a, g) in enumerate(zip(agents, gps)):
        what = f"n={a.n}"
        if not active2[i]:
            assert tuple(rec[i, 3:]) == (0.0, 0.0), what
            continue
        Xf = g.download_X()
        ref, rel = ac.relative_change_ref(Xf, X2[i], a.n)
        assert ref > 0 and abs(ac.LD(rec[i, 3]) - ref) <= rel * ref, (what, rec[i, 3], float(ref))
        assert rec[i, 4] == 1.0, what
        ac.check_status(rec[i], a, Xf, what, G=np.zeros_like(a.G))     # the round's G build cleared the G set earlier


# ---------------------------------------------------------------------------------------------------------------------
# greedy independent-set selection
# ---------------------------------------------------------------------------------------------------------------------
def set_shared(gp, s):
    cp = capi()
    cp.check(lib().dpgo_agent_set_shared_edges(gp._h, len(s.local), cp.iptr(s.local), cp.iptr(s.slot), cp.iptr(s.out),
                                               cp.dptr(s.T), cp.dptr(s.om)))


def check_G(got, s, gathered=None, what="G"):
    ref, bound = s.G_ref(gathered)
    err = abs(ac.ld(got) - ref)
    assert (err <= bound).all(), f"{what}: {int((err > bound).sum())} elements out of bound"
    has = np.zeros(s.n, dtype=bool)
    has[s.local] = True
    assert (sc.tiles(got, s.d)[:, ~has] == 0).all(), f"{what}: a pose without shared edges is not zero"


@pytest.mark.parametrize("k", ac.SELECT_KS)
def test_selection_rounds(k):
    """Crafted records of k agents (ties, +-0, NaN, +inf, subnormals) through dpgo_agents_select_round_async with one real
    agent at the first, middle or last index: every round's mask (read back from the selection log, across its doublings
    for the long runs) equals the host rule; the real agent's iterate and G change only when it is selected."""
    import torch
    L, cp = lib(), capi()
    rounds = 140 if k in (33, 1024) else 12
    idx = (0, k // 2, k - 1)[ac.SELECT_KS.index(k) % 3]
    a = ac.Agent(3, 5, 20, 11)
    gp = handle(a)
    s = ac.SharedEdges(3, 5, 20, seed=k, per_dir=3, slots=8)
    set_shared(gp, s)
    getG = G_reader(gp)
    rng = np.random.default_rng(k)
    gA, gB = s.gathered, rng.standard_normal(s.gathered.shape)
    tA = torch.from_numpy(s.gathered_device_layout(gA)).cuda()
    tB = torch.from_numpy(s.gathered_device_layout(gB)).cuda()
    torch.cuda.synchronize()
    cp.check(L.dpgo_agent_build_G(gp._h, C.c_void_p(tB.data_ptr()), s.slots))
    G_prev = getG()
    check_G(G_prev, s, gB, "G before the rounds")
    ptr, adj = ac.agent_graph(k, ac.graph_kind_for(k))
    adj_arg = adj if len(adj) else np.zeros(1, dtype=np.int32)
    h1 = handles([gp])
    assert L.dpgo_agents_set_agent_graph(gp._h, ac.SELECT_MAX_AGENTS + 1, cp.iptr(np.zeros(1026, dtype=np.int32)),
                                         cp.iptr(adj_arg)) == ERR_INVALID_ARG
    cp.check(L.dpgo_agents_set_agent_graph(gp._h, k, cp.iptr(ptr), cp.iptr(adj_arg)))
    recs = ac.selection_records(k, rounds, seed=k)
    dev = torch.empty(k * ac.STATUS_DOUBLES, dtype=torch.float64, device="cuda")
    prm = params()
    send = (C.c_void_p * 1)(None)
    ai = np.array([idx], dtype=np.int32)
    X_prev, moved, masks = gp.download_X(), 0, []
    for i in range(rounds):
        dev.copy_(torch.from_numpy(np.ascontiguousarray(recs[i]).ravel()))
        torch.cuda.synchronize()
        cp.check(L.dpgo_agents_select_round_async(h1, 1, cp.iptr(ai), C.byref(prm), C.c_void_p(dev.data_ptr()),
                                                  C.c_void_p(tA.data_ptr()), s.slots, send, None))
        gp.sync()
        mask = ac.host_select(recs[i, :, 2], ptr, adj)
        masks.append(mask)
        X, G = gp.download_X(), getG()
        if mask[idx]:
            if moved < 3:                                    # a step from a random start moves X
                assert not np.array_equal(X, X_prev), i
            moved += 1
            check_G(G, s, gA, f"G of round {i}")
        else:
            assert np.array_equal(X, X_prev) and np.array_equal(G, G_prev), i
        X_prev, G_prev = X, G
    log = np.zeros(rounds * k, dtype=np.uint8)
    total = C.c_int64(0)
    cp.check(L.dpgo_agents_selection_log(gp._h, 0, rounds, log.ctypes.data_as(C.POINTER(C.c_uint8)), C.byref(total)))
    assert total.value == rounds
    got = log.reshape(rounds, k)
    for i in range(rounds):
        assert np.array_equal(got[i], masks[i]), (i, np.flatnonzero(got[i] != masks[i])[:8])


# ---------------------------------------------------------------------------------------------------------------------
# G from shared edges
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d,r", DR)
def test_build_G_hub(d, r):
    """a hub pose with 620 shared edges in both directions (interleaved, some duplicated), and edges at the first and
    last pose: G within the per-element bound of constructGMatrix in long double, zero elsewhere, the same bits again"""
    import torch
    cp = capi()
    s = ac.SharedEdges(d, r, 300)
    gp = handle(ac.Agent(d, r, 300, 5))                      # its random G is cleared by the first build
    set_shared(gp, s)
    getG = G_reader(gp)
    t = torch.from_numpy(s.gathered_device_layout()).cuda()
    torch.cuda.synchronize()
    cp.check(lib().dpgo_agent_build_G(gp._h, C.c_void_p(t.data_ptr()), s.slots))
    G = getG()
    check_G(G, s, what=f"G d={d} r={r}")
    cp.check(lib().dpgo_agent_build_G(gp._h, C.c_void_p(t.data_ptr()), s.slots))
    assert np.array_equal(getG(), G)


# ---------------------------------------------------------------------------------------------------------------------
# robust single rotation averaging
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m", ac.ROT_MS)
@pytest.mark.parametrize("d", [2, 3])
def test_rotation_averaging(d, m):
    """1 .. 5000 candidates (past one block of 256 threads), and an all-inlier case that skips GNC: the inlier set and
    GNC iteration count of the CPU restatement, R to 1e-12"""
    cp = capi()
    for all_inlier in ((False, True) if m == 1000 else (False,)):
        R = np.ascontiguousarray(ac.rotation_inputs(d, m, all_inlier), dtype=np.float64)
        Ro, inl, its, _ = dio.robust_single_rotation_averaging(R, cbar=dio.CBAR)
        out = np.zeros((d, d))
        flags = np.zeros(m, dtype=np.int32)
        its_g = C.c_int32(-1)
        cp.check(lib().dpgo_robust_single_rotation_averaging(0, d, m, cp.dptr(R), None, dio.CBAR, cp.dptr(out),
                                                             cp.iptr(flags), C.byref(its_g)))
        what = (d, m, all_inlier)
        assert [int(i) for i in np.flatnonzero(flags)] == inl and its_g.value == its, what
        assert np.abs(out - Ro).max() <= 1e-12, what
        if ac.gnc_skipped(R, dio.CBAR):
            assert its == 0 and len(inl) == m, what
        else:
            assert its > 0 and 0 < len(inl) < m, what


# ---------------------------------------------------------------------------------------------------------------------
# a handle listed twice
# ---------------------------------------------------------------------------------------------------------------------
def test_duplicate_handles_refused():
    """The seven batched calls refuse one handle listed twice (two jobs would share its ticket counter, or write its
    alignment buffers and X at once) and enqueue nothing: the agent's iterate is unchanged and its next status record is
    bitwise the one before, so its ticket was not touched."""
    import torch
    L, cp = lib(), capi()
    a = ac.Agent(3, 5, 1100, 3)                              # 35 status CTAs
    gp = handle(a)
    T = np.asfortranarray(np.tile(np.hstack([np.eye(3), np.zeros((3, 1))]), (1, a.n)))
    Y = np.asfortranarray(orc.fixed_stiefel_variable(3, 5))
    # the align call's state is set, so only the duplicate can refuse it; X = Y T is then undone
    cp.check(L.dpgo_agent_set_local_trajectory(gp._h, cp.dptr(T), cp.dptr(Y)))
    cp.check(L.dpgo_agent_set_align_candidates(gp._h, 0, None, None, None, None, None, None))
    gp.upload_X(a.X)
    pub = np.arange(4, dtype=np.int32)
    cp.check(L.dpgo_agent_set_public_poses(gp._h, len(pub), cp.iptr(pub)))
    cp.check(L.dpgo_agent_accel_init(gp._h))
    before = status([gp], [0], 1)[0]
    ac.check_status(before, a, a.X, "before")
    two = handles([gp, gp])
    idx2 = np.array([0, 1], dtype=np.int32)
    buf = nan_tensor(2 * ac.STATUS_DOUBLES)
    send = [nan_tensor(4 * 20) for _ in range(2)]
    prm = params()
    assert L.dpgo_agents_status_async(two, 2, cp.iptr(idx2), C.c_void_p(buf.data_ptr()), None) == ERR_INVALID_ARG
    assert L.dpgo_agents_accel_begin_async(two, 2, cp.iptr(np.ones(2, dtype=np.int32)), 5.0, 30, ptrs(send), ptrs(send),
                                           None) == ERR_INVALID_ARG
    assert L.dpgo_agents_round_async(two, 2, C.byref(prm), None, 0, ptrs(send), None, 0) == ERR_INVALID_ARG
    assert L.dpgo_agents_accel_round_async(two, 2, C.byref(prm), None, None, 0, None) == ERR_INVALID_ARG
    ptr, adj = ac.agent_graph(2, "path")
    cp.check(L.dpgo_agents_set_agent_graph(gp._h, 2, cp.iptr(ptr), cp.iptr(adj)))
    assert L.dpgo_agents_select_round_async(two, 2, cp.iptr(idx2), C.byref(prm), C.c_void_p(buf.data_ptr()), None, 0,
                                            ptrs(send), None) == ERR_INVALID_ARG
    zeros = [np.zeros(a.r * (a.d + 1) * a.n) for _ in range(2)]          # an upload of either would change X
    X_host = (C.c_void_p * 2)(*[z.ctypes.data for z in zeros])
    assert L.dpgo_agents_host_io_async(two, 2, X_host, None, 0, None) == ERR_INVALID_ARG
    assert L.dpgo_agents_align_async(two, 2, None, 0, cp.iptr(np.ones(1, dtype=np.int32)), 1, None) == ERR_INVALID_ARG
    torch.cuda.synchronize()
    assert np.isnan(buf.cpu().numpy()).all()
    assert np.array_equal(gp.download_X(), a.X)
    assert np.array_equal(status([gp], [0], 1)[0], before)

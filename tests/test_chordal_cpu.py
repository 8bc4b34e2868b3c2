"""The chordal-initialisation reference of chordal_reference.py against the oracle and known answers, and the argument
checks of dpgo_chordal_initialization, which all run before any device call (no GPU needed)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import chordal_reference as cr  # noqa: E402
import structure_cases as sc  # noqa: E402
from oracle import dpgo_oracle as orc  # noqa: E402

ERR_INVALID_ARG = 1          # DPGO_ERR_INVALID_ARG of include/dpgo_b200.h


@pytest.mark.parametrize("ds", ["tinyGrid3D", "smallGrid3D", "CSAIL", "input_INTEL_g2o"])
def test_reference_matches_oracle(ds, data_dir):
    from dpo_b200 import posegraph as pg
    path = os.path.join(data_dir, ds + ".g2o")
    edges, n = pg.read_g2o_file(path)
    meas, _ = orc.read_g2o(path)
    ref = cr.chordal_reference(edges, n)
    To = orc.chordal_initialization(meas, n)
    assert np.abs(ref.T() - To).max() <= 1e-10 * max(1.0, np.abs(To).max())
    assert ref.rot.refined_to <= 1e-17 and ref.tra.refined_to <= 1e-17


@pytest.mark.parametrize("graph,d", [("chain", 2), ("chain", 3), ("grid", 3)])
def test_reference_matches_noise_free_known_answer(graph, d):
    """A noise-free graph's least-squares problems have the ground truth (in the gauge of pose 0) as exact solution."""
    if graph == "chain":
        n, edges, Tgt = sc.noise_free_graph(d, sc.chain(range(300)), 300, seed=1)
    else:
        from dpo_b200 import posegraph as pg
        edges, n, Tgt = pg.synthetic_grid_graph(6, 6, 4, seed=1, rot_sigma=0.0, trans_sigma=0.0)
    ref = cr.chordal_reference(edges, n)
    expect = sc.in_gauge_of_pose_zero(Tgt, d)
    assert np.abs(ref.T() - expect).max() <= 1e-11 * max(1.0, np.abs(expect).max())


def test_reference_components_and_isolated_poses():
    """Outside the component of pose 0 the reference keeps R = I and t = 0; the component's rotations are unprojected
    least-squares solutions with zero gradient there."""
    case = sc.make_case("components", 3)
    ref = cr.chordal_reference(case.edges, case.n)
    comp = cr.component_of_zero(case.n, case.edges.p1, case.edges.p2, case.edges.kappa)
    assert comp.sum() == 30
    assert np.array_equal(ref.R[~comp], np.broadcast_to(np.eye(3), (int((~comp).sum()), 3, 3)))
    assert np.all(ref.t[~comp] == 0)
    x = cr.ld(ref.M).transpose(0, 2, 1).reshape(-1)
    b, bm = ref.rot.rhs()
    assert float(np.max(np.abs(b - ref.rot.apply(x)))) <= 1e-15 * float(np.max(bm))


# ---- argument checks of dpgo_chordal_initialization --------------------------------------------------------------
def _call(n, d, m, p1, p2, R, t, kap, tau, T, its=None):
    from dpo_b200 import _capi as capi
    lib = capi.load_library()
    ptr = lambda a, f: None if a is None else f(a)
    code = lib.dpgo_chordal_initialization(n, d, m, ptr(p1, capi.iptr), ptr(p2, capi.iptr), ptr(R, capi.dptr), ptr(t, capi.dptr),
                                           ptr(kap, capi.dptr), ptr(tau, capi.dptr), 0, 0.0, 0, ptr(T, capi.dptr), its)
    return code, lib.dpgo_chordal_last_error().decode()


def _arrays(d, m, n):
    rng = np.random.default_rng(0)
    e = sc.edge_set(rng, d, sc.chain(range(m + 1)))
    return (np.ascontiguousarray(e.p1, dtype=np.int32), np.ascontiguousarray(e.p2, dtype=np.int32),
            np.ascontiguousarray(e.R), np.ascontiguousarray(e.t), e.kappa.copy(), e.tau.copy(),
            np.zeros((d, (d + 1) * n), order="F"))


@pytest.mark.parametrize("what", ["n<1", "d=4", "d=1", "m<0", "null p1", "null p2", "null R", "null t", "null kappa",
                                  "null tau", "p1 out of range", "p2 negative", "null T"])
def test_argument_errors(what):
    d, m, n = 3, 4, 5
    p1, p2, R, t, kap, tau, T = _arrays(d, m, n)
    args = dict(n=n, d=d, m=m, p1=p1, p2=p2, R=R, t=t, kap=kap, tau=tau, T=T)
    if what == "n<1":
        args["n"] = 0
    elif what == "d=4":
        args["d"] = 4
    elif what == "d=1":
        args["d"] = 1
    elif what == "m<0":
        args["m"] = -1
    elif what.startswith("null "):
        args[{"kappa": "kap"}.get(what[5:], what[5:])] = None
    elif what == "p1 out of range":
        p1[2] = n
    elif what == "p2 negative":
        p2[1] = -1
    T0 = T.copy()
    code, msg = _call(**args)
    assert code == ERR_INVALID_ARG and msg
    if args["T"] is not None:
        assert np.array_equal(T, T0)


@pytest.mark.parametrize("d", [2, 3])
def test_single_pose_is_the_gauge(d):
    """n = 1: [I | 0] and no CG iteration (no device call is made)."""
    from dpo_b200 import _capi as capi
    T = np.full((d, d + 1), 7.0, order="F")
    its = (C.c_int32 * 2)(5, 5)
    code, msg = _call(1, d, 0, None, None, None, None, None, None, T, its)
    assert code == capi.OK, msg
    assert np.array_equal(T, np.hstack([np.eye(d), np.zeros((d, 1))])) and list(its) == [0, 0]

"""CPU checks of the edge-record cases and references of edge_cases.py:

  * every case reaches what it is built for, from host facts only;
  * the long-double Q reference agrees with the oracle's connection Laplacian on four datasets, and the exact read-back
    of Q through selector rows of X Q returns Q bit for bit;
  * reference_weight restates RobustCost::weight (ref src/DPGO_robust.cpp:23-66), and the host port computes it bit for bit;
  * the device formula before the fix (r^2 in place of sqrt(r^2)^2, the bounds in another order) puts crafted boundary
    residuals in another GNC class than the reference."""
import math
import os
import subprocess

import numpy as np
import pytest

import edge_cases as ec
from oracle import dpgo_oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALL = [(name, d) for name in ec.CASE_NAMES for d in (2, 3)]


@pytest.fixture(scope="module")
def cases():
    return {}


def get(cases, name, d):
    if (name, d) not in cases:
        cases[(name, d)] = ec.make_case(name, d)
    return cases[(name, d)]


@pytest.mark.parametrize("name,d", ALL)
def test_case_reaches_its_target(name, d, cases):
    c = get(cases, name, d)
    e = c.edges
    m = len(e)
    ns = 0 if c.static_pose is None else len(c.static_pose)
    edge_poses = set(e.p1.tolist()) | set(e.p2.tolist())
    assert c.target
    if name != "path1e6":
        qref = ec.q_reference(c)
    if name == "static_only":
        assert (c.n, m, ns) == (1, 0, 1) and list(qref) == [(0, 0)]
    elif name == "no_edges":
        assert c.n > 1 and m == 0 and ns == 0 and qref == {}
    elif name == "static_on_edge_pose":
        assert ns == 1 and int(c.static_pose[0]) in edge_poses
    elif name == "static_on_free_pose":
        p = int(c.static_pose[0])
        assert ns == 1 and p not in edge_poses and qref[(p, p)][2] == 1
    elif name == "static_twice":
        assert len(set(c.static_pose.tolist())) < ns
    elif name == "static_nonsymmetric":
        S = c.static_blocks[0]
        assert np.abs(S - S.T).max() > 0.1
    elif name == "star2100":
        assert qref[(0, 0)][2] == ec.HUB_LEAVES and (e.p1 == 0).any() and (e.p2 == 0).any()
    elif name == "clique60":
        assert len(qref) == c.n * c.n
    elif name == "repeated_pair":
        fwd, bwd = ((e.p1 == 0) & (e.p2 == 1)).sum(), ((e.p1 == 1) & (e.p2 == 0)).sum()
        assert fwd == bwd == 50 and qref[(0, 1)][2] == 100
    elif name == "wide_weights":
        w = e.weight[e.weight > 0]
        assert (e.weight == 0).sum() >= 3 and np.log10(w.max() / w.min()) > 150
        assert set(ec.zero_only_poses(c).tolist()) == set(range(40, 45))
    elif name == "wide_kappa_tau":
        for v in (e.kappa, e.tau):
            assert np.log10(v.max() / v.min()) > 12
    elif name == "non_orthonormal":
        gram = np.einsum("mba,mbc->mac", e.R, e.R)
        assert np.abs(gram - np.eye(d)).max() > 0.5 and np.abs(e.t).max() == 1e6
    elif name == "path1e6":
        assert m == 10 ** 6 and c.fixed.sum() == (m + 6) // 7


@pytest.mark.parametrize("ds", ["tinyGrid3D", "smallGrid3D", "CSAIL", "input_INTEL_g2o"])
def test_q_reference_agrees_with_oracle(ds, data_dir):
    from dpo_b200 import posegraph as pg
    edges, n = pg.read_g2o_file(os.path.join(data_dir, ds + ".g2o"))
    meas, _ = orc.read_g2o(os.path.join(data_dir, ds + ".g2o"))
    rng = np.random.default_rng(3)
    w = rng.uniform(0.1, 2.0, len(edges))
    edges.weight, meas.weight = w.copy(), w.copy()
    c = ec.EdgeCase(ds, edges.d, n, edges, "dataset")
    Q = orc.construct_connection_laplacian(meas, n).tocsr()
    qref = ec.q_reference(c)
    dh = c.dh
    blocks = {(i, j): Q[i * dh:(i + 1) * dh, j * dh:(j + 1) * dh].toarray() for (i, j) in qref}
    assert np.isclose(sum(abs(B).sum() for B in blocks.values()), abs(Q).sum(), rtol=1e-12, atol=0)    # nothing outside
    ec.check_q(blocks, qref, ds)
    # the bound has power: 1e-12 of relative error in one diagonal entry is out of it
    i = int(edges.p1[5])
    bad = dict(blocks)
    bad[(i, i)] = bad[(i, i)].copy()
    bad[(i, i)][0, 0] *= 1.0 + 1e-12
    with pytest.raises(AssertionError):
        ec.check_q(bad, qref)


@pytest.mark.parametrize("name,d", [(n, d) for n in ec.READBACK for d in (2, 3)])
def test_selector_read_back_is_exact(name, d, cases):
    """read_back through a float64 X Q returns the host-summed Q bit for bit: each output entry is one product by 1.0"""
    c = get(cases, name, d)
    Q = c.Q()
    got = ec.read_back(lambda X: np.asarray((Q.T @ X.T).T), c, 8)
    Qb = Q.toarray() if c.N else np.zeros((0, 0))
    assert set(got) == set(ec.q_reference(c))
    for (i, j), B in got.items():
        assert np.array_equal(B, Qb[i * c.dh:(i + 1) * c.dh, j * c.dh:(j + 1) * c.dh]), (i, j)
    classes, _ = ec.selector_classes(c)
    if name == "star2100":
        assert len(classes) == c.n                    # every leaf shares the hub's column: one pose per class


# ---------------------------------------------------------------------------------------------------------------------
# weights
# ---------------------------------------------------------------------------------------------------------------------
def scalar_weight(cost, r, mu, c, fused_gm=False):
    """RobustCost::weight(r) transcribed line by line in Python floats (IEEE double, correctly rounded operations)"""
    if cost == "L2":
        return 1.0
    if cost == "L1":
        return 1.0 / r if r != 0 else math.inf
    if cost == "Huber":
        return 1.0 if r < c else (c / r if r != 0 else math.nan)
    if cost == "TLS":
        return 1.0 if r < c else 0.0
    if cost == "GM":
        a = float(ec.Fraction(r) ** 2 + 1) if fused_gm else 1 + r * r
        return 1 / (a * a)
    rSq = r * r
    mGNCBarcSq = c * c
    upperBound = (mu + 1) / mu * mGNCBarcSq
    lowerBound = mu / (mu + 1) * mGNCBarcSq
    if rSq >= upperBound:
        return 0.0
    if rSq <= lowerBound:
        return 1.0
    return math.sqrt(mGNCBarcSq * mu * (mu + 1) / rSq) - mu


def crafted_probes():
    """(cost, r2, mu, c): the GNC boundary set, Huber / TLS thresholds, r = 0, and random r2 over many decades"""
    rng = np.random.default_rng(9)
    out = [("GNC_TLS", v, mu, c) for mu, c, v in ec.gnc_boundary_set()]
    for cost in ("Huber", "TLS"):
        for c in (0.5, 3.0, 10.0, 1e-3):
            out += [(cost, float(v), 1.0, c) for v in ec.boundary_probes(cost, 1.0, c)]
    r2 = np.concatenate([[0.0], 10.0 ** rng.uniform(-12, 12, 400)])
    for cost in ec.COSTS:
        for mu in (1e-4, 0.3, 2.0):
            out += [(cost, float(v), mu, 3.0) for v in r2]
    return out


def same(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return (a == b) | (np.isnan(a) & np.isnan(b))


def test_reference_weight_restates_the_reference():
    probes = crafted_probes()
    for gm in ("separate", "fused"):
        for cost, r2, mu, c in probes:
            got = ec.reference_weight(cost, r2, mu, c, gm=gm)
            want = scalar_weight(cost, math.sqrt(r2), mu, c, fused_gm=(gm == "fused"))
            assert same(got, want), (cost, r2, mu, c, gm, float(got), want)
    # vectorised over r2 as the GPU tests call it
    r2 = np.array([p[1] for p in probes if p[0] == "GM"])
    assert same(ec.reference_weight("GM", r2), [scalar_weight("GM", math.sqrt(v), 1, 1) for v in r2]).all()
    # the two GM variants differ (so the variant the device matches is a real choice), GNC has one value
    gm = [p for p in probes if p[0] == "GM"]
    diff = sum(not same(ec.reference_weight("GM", v, gm="separate"), ec.reference_weight("GM", v, gm="fused")) for _, v, _, _ in gm)
    assert diff > 0
    assert ec.reference_weight("L1", 0.0) == np.inf                                   # 1 / r at r = 0, as the reference
    assert ec.reference_weight("GNC_TLS", 0.0, 1e-4, 0.0) == 0.0                       # barc = 0: every residual rejected


def test_prefix_device_formula_misclassifies_boundary_residuals():
    """the device formula before the fix puts some crafted GNC residuals in another class (1 / 0 / in between) than the
    reference's, so its counts stopped GNC in another round; GM from 1 + r2 differs in the last bits"""
    wrong = 0
    for mu, c, v in ec.gnc_boundary_set():
        if ec.classify(ec.prefix_device_weight("GNC_TLS", v, mu, c)) != ec.classify(ec.reference_weight("GNC_TLS", v, mu, c)):
            wrong += 1
    assert wrong > 0
    rng = np.random.default_rng(4)
    r2 = 10.0 ** rng.uniform(-3, 3, 2000)
    assert (ec.prefix_device_weight("GM", r2) != ec.reference_weight("GM", r2)).any()


@pytest.fixture(scope="module")
def host_check():
    from dpo_b200 import build
    return build.build_cpp_program([os.path.join(ROOT, "tests", "cpp", "host_check.cpp")],
                                   os.path.join(ROOT, "build", "tests", "host_check"))


def test_host_port_weights_are_the_reference_bit_for_bit(host_check, tmp_path):
    probes = crafted_probes()
    path = tmp_path / "probes.txt"
    with open(path, "w") as fh:
        for cost, r2, mu, c in probes:
            fh.write(f"{cost} {math.sqrt(r2).hex()} {float(mu).hex()} {float(c).hex()}\n")
    res = subprocess.run([host_check, "--weights", str(path)], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-2000:]
    got = [float.fromhex(ln.split()[1].replace("-nan", "nan")) for ln in res.stdout.splitlines() if ln.startswith("weight")]
    assert len(got) == len(probes)
    for (cost, r2, mu, c), w in zip(probes, got):
        assert same(w, ec.reference_weight(cost, r2, mu, c)), (cost, r2, mu, c, w, float(ec.reference_weight(cost, r2, mu, c)))

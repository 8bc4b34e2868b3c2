"""One small dpgo_pose_covariances call per model (SE(3) with pairs, SE(2)), for the compute-sanitizer memcheck run of
tests/test_gpu_covariance.py.  Prints "ok" when both calls return."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from dpo_b200 import posegraph as pg  # noqa: E402

edges, n = pg.read_g2o_file(os.path.join(ROOT, "data", "tinyGrid3D.g2o"))
T = pg.chordalInitialization(3, n, edges)
cov, pcov = pg.poseCovariancesGPU(edges, n, T, anchor=1, pairs=[[0, n - 1], [2, 3], [4, 4]])
assert np.all(np.isfinite(cov)) and np.all(np.isfinite(pcov))
edges2, n2 = pg.read_g2o_file(os.path.join(ROOT, "data", "input_INTEL_g2o.g2o"))
keep = np.nonzero((edges2.p1 < 200) & (edges2.p2 < 200))[0]
e2 = edges2.take(keep)
T2 = pg.chordalInitialization(2, 200, e2)
cov2 = pg.poseCovariancesGPU(e2, 200, T2, pairs=[[3, 150]])[0]
assert np.all(np.isfinite(cov2))
# a 2D star anchored at its hub: non-root macro nodes whose boundary is empty, so the sweep runs no product
sys.path.insert(0, os.path.join(ROOT, "tests"))
import covariance_cases as cc  # noqa: E402
hub = cc.make_case("hub2100_anchor_hub", 2)
code, cov3, _, info3 = cc.call_device(hub)
assert code == 0 and info3[6] == 0 and info3[1] > 1 and np.all(np.isfinite(cov3))
print("ok")

"""One RTR step at r = 8 with the exact preconditioner in each launch mode (full grid, one thread-block cluster), for the
compute-sanitizer memcheck run of tests/test_gpu_ranks.py.  Prints "ok" when both steps return."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import dpo_b200 as dp  # noqa: E402
from dpo_b200 import posegraph as pg  # noqa: E402

edges, n = pg.read_g2o_file(os.path.join(ROOT, "data", "tinyGrid3D.g2o"))
r = 8
X0 = pg.fixedStiefelVariable(3, r) @ pg.chordalInitialization(3, n, edges)
for cluster in (False, True):
    gp = dp.QuadraticProblem(n, 3, r, cluster=cluster)
    gp.setQ_blocks(*pg.connection_laplacian_blocks(edges))
    go = dp.QuadraticOptimizer(gp)
    go.setTrustRegionIterations(1)
    go.setTrustRegionMaxInnerIterations(10)
    X = go.optimize(X0)
    assert go.getOptResult().success == 1 and np.all(np.isfinite(X))
    gp.close()
print("ok")

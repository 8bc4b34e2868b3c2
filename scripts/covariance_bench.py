"""Timing of the pose covariances on the GPU (dpgo_pose_covariances): assembly of the Gauss-Newton information, its
factorisation and the selected-inversion sweep, per dataset, from device events around each part (info16[10..12]).

    python scripts/covariance_bench.py [--reps 5] [datasets...]

Prints the device, its power limit and SM clock, then one line per dataset: the hierarchy (macro levels, nodes, largest
own / boundary block, device bytes) and the median of each part over the repetitions.  The trajectory is the chordal
initialisation (CPU)."""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from dpo_b200 import posegraph as pg  # noqa: E402


def device_line():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out.splitlines()[0] if out else "nvidia-smi: no output"
    except Exception as e:              # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("datasets", nargs="*", default=["sphere2500", "torus3D", "grid3D", "city10000"])
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    print("device (name, power limit, SM clock, max SM clock):", device_line())
    for name in a.datasets:
        edges, n = pg.read_g2o_file(os.path.join(ROOT, "data", name + ".g2o"))
        T = pg.chordalInitialization(edges.d, n, edges)
        pg.poseCovariancesGPU(edges, n, T)                     # warm-up: module load, first allocations
        times = []
        for _ in range(a.reps):
            _, info = pg.poseCovariancesGPU(edges, n, T, return_info=True)
            times.append(info[10:13])
        med = np.median(np.array(times, dtype=np.float64), axis=0) / 1e6
        print(f"{name}: n={n} d={edges.d} levels={info[0]} nodes={info[1]} own<={info[5]} bnd<={info[6]} "
              f"bytes={info[4] / 1e6:.1f}MB | assembly {med[0]:.3f} ms  factor {med[1]:.3f} ms  sweep {med[2]:.3f} ms "
              f"(median of {a.reps})", flush=True)


if __name__ == "__main__":
    main()

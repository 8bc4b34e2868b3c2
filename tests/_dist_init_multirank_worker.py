"""Worker of tests/test_gpu_dist_init.py: one rank of a torchrun launch.  Builds the distributed start of a k-agent split
with the agents spread over the ranks (local chordal solves on each rank, public tiles and per-wave outcomes by NCCL
all-gather) and writes this rank's iterates and the initialisation report."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ds, k, out_dir = sys.argv[1], int(sys.argv[2]), sys.argv[3]
    import torch
    import torch.distributed as dist
    from dpo_b200 import posegraph as pg
    from dpo_b200.agent import DistributedPGO
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    edges, n = pg.read_g2o_file(os.path.join(ROOT, "data", ds + ".g2o"))
    run = DistributedPGO(edges, n, k, r=5, schedule="coloured", rank=rank, world=world, device=local, dist=dist,
                         concurrent=False, initialization="distributed")
    for a in run.local_ids:
        np.save(os.path.join(out_dir, f"X_{a}.npy"), run.agents[a].mProblem.download_X())
    if rank == 0:
        with open(os.path.join(out_dir, "report.json"), "w") as fh:
            json.dump(run.init_report, fh)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()

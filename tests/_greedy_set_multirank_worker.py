"""Worker of tests/test_gpu_greedy_set.py: one rank of a torchrun launch.  Runs `rounds` greedy_set rounds of the k-agent
split with the agents spread over the ranks (status records and public poses by NCCL all-gather) and writes this rank's
iterates and its selection log."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ds, k, rounds, out_dir, conc = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), sys.argv[4], int(sys.argv[5])
    import torch
    import torch.distributed as dist
    from dpo_b200 import posegraph as pg
    from dpo_b200.agent import DistributedPGO
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    edges, n = pg.read_g2o_file(os.path.join(ROOT, "data", ds + ".g2o"))
    run = DistributedPGO(edges, n, k, r=5, schedule="greedy_set", rank=rank, world=world, device=local, dist=dist,
                         concurrent=bool(conc))
    for _ in range(rounds):
        run.step(evaluate=False)
    for a in run.local_ids:
        np.save(os.path.join(out_dir, f"X_{a}.npy"), run.agents[a].mProblem.download_X())
    log = np.zeros((rounds, k), dtype=np.uint8)
    for i, s in enumerate(run.selection_log()):
        log[i, s] = 1
    np.save(os.path.join(out_dir, f"log_{rank}.npy"), log)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()

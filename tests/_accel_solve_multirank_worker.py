"""Worker of tests/test_gpu_accel_solve.py::test_two_rank_accelerated_solve_bit_equal_to_one_process: one rank of a
torchrun launch.  Runs DistributedPGO.solve with colour-momentum accelerated rounds on the k-agent coloured split, agents
spread over the ranks and the launch mode pinned, and writes this rank's iterates, the report and the gathered records."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ds, k, conc, check_every, out_dir = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4]), sys.argv[5]
    import torch
    import torch.distributed as dist
    from dpo_b200 import posegraph as pg
    from dpo_b200.agent import DistributedPGO
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    edges, n = pg.read_g2o_file(os.path.join(ROOT, "data", ds + ".g2o"))
    run = DistributedPGO(edges, n, k, r=5, schedule="coloured", rank=rank, world=world, device=local, dist=dist,
                         acceleration=True, momentum_blocks="colours", concurrent=bool(conc))
    rep = run.solve(gradnorm_tol=0.1, rel_change_tol=5e-3, check_every=check_every)
    records = run.status().records
    for a in run.local_ids:
        np.save(os.path.join(out_dir, f"X_{a}.npy"), run.agents[a].mProblem.download_X())
    if rank == 0:
        np.save(os.path.join(out_dir, "records.npy"), records)
        np.save(os.path.join(out_dir, "report.npy"), np.array([rep.rounds, rep.cost, rep.gradnorm]))
        with open(os.path.join(out_dir, "reason.txt"), "w") as fh:
            fh.write(rep.reason)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()

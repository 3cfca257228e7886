"""torchrun worker of tests/test_lbfgs_gpu.py::test_data_parallel_ranks_end_with_identical_theta (one rank per GPU).

  python -m torch.distributed.run --nproc-per-node 2 ... tests/dp_lbfgs_worker.py <workload> <out.json>

Every rank fits the same problem with FlatLBFGS under data parallelism (each closure all-reduces [grad | sum r^2]);
rank 0 writes whether the ranks' parameters are bit-identical."""
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    key, out = sys.argv[1], sys.argv[2]
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    from neurodiffeq_b200.optim import FlatLBFGS
    from test_solvers_gpu import make_solver

    wl, solver, nets, _ = make_solver(key, 3001)
    assert solver._dist is not None
    solver.optimizer = FlatLBFGS.for_solver(solver, lr=0.5, max_iter=4, history_size=5)
    solver.fit(3, tqdm_file=None)
    theta = solver.problem.theta.clone()
    gathered = [torch.empty_like(theta) for _ in range(world)]
    dist.all_gather(gathered, theta)
    identical = all(bool(torch.equal(g, gathered[0])) for g in gathered)
    dist.barrier()
    if rank == 0:
        with open(out, "w") as f:
            json.dump({"workload": key, "world": world, "identical": identical,
                       "losses": solver.metrics_history["train_loss"]}, f)
    torch.cuda.synchronize()
    dist.barrier()
    sys.stdout.flush()
    os._exit(0)     # skip the NCCL teardown


if __name__ == "__main__":
    main()

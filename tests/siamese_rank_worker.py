"""Worker of tests/test_siamese_e2e_gpu.py::test_siamese_two_ranks_equal_one_rank (one process per GPU under torch.distributed.run):
the siamese-shaped net of tests/test_siamese_sim.py, every tower blob shared by name, trained with SGD through the C++ TrainNet +
P2PSync + ReduceScheduler on this rank's slice of the global batch; dumps parameters and momentum to <outdir>/rank<r>.npz."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def run(trainer_batch, params, data, label, steps, sync=None):
    import test_siamese_sim as ss
    from caffe_mpi_b200 import host_api
    t = host_api.Trainer(ss.net(trainer_batch), ss.SOLVER, num_classes=ss.CLS)
    for i, p in enumerate(params):
        t.set_param(i, p)
    if sync is not None:
        world, rank, dist = sync
        ids = [t.new_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(ids, src=0)
        t.attach_sync(world, rank, ids[0])
    t.set_blob("pair_data", data)
    t.set_blob("label", label)
    for _ in range(steps):
        t.step(1)
    t.sync()
    return {f"{n}{i}": t.get_param(i, k) for i in range(len(params)) for n, k in (("p", 0), ("h", 2))}


def main():
    import torch
    import torch.distributed as dist
    import test_siamese_sim as ss
    outdir, global_batch, steps = sys.argv[1], int(sys.argv[2]), int(sys.argv[3])
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("gloo")
    params, data, label = ss.case(global_batch, seed=13)
    per = global_batch // world
    sl = slice(rank * per, (rank + 1) * per)
    np.savez(os.path.join(outdir, f"rank{rank}.npz"), **run(per, params, data[sl], label[sl], steps, sync=(world, rank, dist)))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()

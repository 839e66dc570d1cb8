"""Worker of tests/test_clip_gpu.py::test_two_gpus_equal_one (one process per GPU under torch.distributed.run): LeNet trained with SGD
and clip_gradients through the C++ TrainNet + P2PSync + ReduceScheduler on this rank's slice of multi_rank_worker.build_case's global
batch; dumps this rank's parameters, history and clipped-step count to <outdir>/rank<r>.npz."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

SOLVER = 'type: "SGD" base_lr: 0.05 lr_policy: "fixed" momentum: 0.9 weight_decay: 0.0005 max_iter: 100 clip_gradients: 0.5'


def run(trainer_batch, params, data, label, steps, sync=None):
    import netoracle as no
    from caffe_mpi_b200 import host_api
    t = host_api.Trainer(no.to_prototxt(no.lenet(batch=trainer_batch)), SOLVER, num_classes=10)
    for i, p in enumerate(params):
        t.set_param(i, p)
    if sync is not None:
        world, rank, dist = sync
        ids = [t.new_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(ids, src=0)
        t.attach_sync(world, rank, ids[0])
    t.set_blob("data", data)
    t.set_blob("label", label)
    for _ in range(steps):
        t.step(1)
    t.sync()
    out = {f"{n}{i}": t.get_param(i, k) for i in range(len(params)) for n, k in (("p", 0), ("h", 2))}
    out["clipped"] = np.array(t.clip_state()[2])
    return out


def main():
    import torch
    import torch.distributed as dist
    import multi_rank_worker as mw
    outdir, global_batch, steps = sys.argv[1], int(sys.argv[2]), int(sys.argv[3])
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("gloo")
    params, data, label = mw.build_case(global_batch)
    per = global_batch // world
    sl = slice(rank * per, (rank + 1) * per)
    np.savez(os.path.join(outdir, f"rank{rank}.npz"), **run(per, params, data[sl], label[sl], steps, sync=(world, rank, dist)))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()

"""Worker of tests/test_neuron_e2e_gpu.py::test_two_ranks_end_with_bitwise_equal_slopes (one process per GPU under
torch.distributed.run): the neuron net of tests/neuron_oracle.py (in-place PReLU, per-channel or channel-shared slope) trained with
SGD through the C++ TrainNet + P2PSync + ReduceScheduler on this rank's slice of the global batch; dumps the parameters to
<outdir>/rank<r>.npz."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

H, W, CLS = 6, 5, 3
SOLVER = 'base_lr: 0.05 lr_policy: "fixed" momentum: 0.9 max_iter: 10'


def case(global_batch, shared, seed=13):
    import neuron_oracle as no
    rng = np.random.default_rng(seed)
    params = []
    for i, sh in enumerate(no.net_param_shapes(H, W, CLS, shared)):
        sh = sh if sh else (1,)
        if i == 2:
            params.append(rng.uniform(0.1, 0.4, sh).astype(np.float32))
        else:
            fan = int(np.prod(sh[1:])) if len(sh) > 1 else 1
            params.append((rng.standard_normal(sh) * (0.5 / np.sqrt(fan))).astype(np.float32))
    data = rng.standard_normal((global_batch, 3, H, W)).astype(np.float32)
    label = rng.integers(0, CLS, global_batch).astype(np.float32)
    return params, data, label


def run(trainer_batch, params, data, label, steps, shared, sync=None):
    import neuron_oracle as no
    from caffe_mpi_b200 import host_api
    t = host_api.Trainer(no.net_prototxt(trainer_batch, H, W, CLS, shared), SOLVER, num_classes=CLS)
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
    return {f"p{i}": t.get_param(i, 0) for i in range(len(params))}


def main():
    import torch
    import torch.distributed as dist
    outdir, global_batch, steps, shared = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), bool(int(sys.argv[4]))
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("gloo")
    params, data, label = case(global_batch, shared)
    per = global_batch // world
    sl = slice(rank * per, (rank + 1) * per)
    np.savez(os.path.join(outdir, f"rank{rank}.npz"), **run(per, params, data[sl], label[sl], steps, shared, sync=(world, rank, dist)))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()

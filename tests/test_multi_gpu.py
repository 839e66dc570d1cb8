"""Multi-GPU correctness on hardware (needs >= 2 GPUs): N data-parallel solvers over the C++
P2PSync / ReduceScheduler are equivalent to one solver on the concatenated batch -- the reference's own check
(src/caffe/test/test_gradient_based_solver.cpp:471-509 runs every solver test with several devices and compares against the
single-device update; parallel.cpp:208-253 and net.cpp:880-912 are the paths exercised)."""
import os
import socket
import subprocess
import sys
import tempfile

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def rel(a, b):
    return float(np.abs(a.astype(np.float64) - b.astype(np.float64)).max() / max(float(np.abs(b).max()), 1e-20))


@pytest.mark.parametrize("world", [2, 4])
def test_n_ranks_equal_one_rank_on_the_full_batch(world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    import multi_rank_worker as mw
    global_batch, steps = 64, 3
    with tempfile.TemporaryDirectory() as td:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
               "--master-port", str(free_port()), os.path.join(ROOT, "tests", "multi_rank_worker.py"), td, str(global_batch), str(steps)]
        r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-4000:])
        ranks = [dict(np.load(os.path.join(td, f"rank{i}.npz"))) for i in range(world)]
    params, data, label = mw.build_case(global_batch)
    one = mw.run(global_batch, params, data, label, steps)                    # one solver, the whole batch, this process
    n = len(params)
    for i in range(n):
        for rk in ranks[1:]:                                                    # (a) every rank holds the same bits
            assert np.array_equal(ranks[0][f"p{i}"].view(np.uint32), rk[f"p{i}"].view(np.uint32)), f"param {i} differs across ranks"
            assert np.array_equal(ranks[0][f"h{i}"].view(np.uint32), rk[f"h{i}"].view(np.uint32)), f"history {i} differs across ranks"
        assert rel(ranks[0][f"p{i}"], one[f"p{i}"]) < 1e-5, (i, rel(ranks[0][f"p{i}"], one[f"p{i}"]))     # (b) == 1 rank, full batch
        hfloor = 1e-3 * max(float(np.abs(one[f"h{j}"]).max()) for j in range(n))
        assert float(np.abs(ranks[0][f"h{i}"] - one[f"h{i}"]).max()) / max(float(np.abs(one[f"h{i}"]).max()), hfloor) < 1e-4, i
    # the global loss is the mean of the per-rank losses (each normalised by its own batch)
    mean_loss = np.mean([rk["losses"] for rk in ranks], axis=0)
    np.testing.assert_allclose(mean_loss, one["losses"], rtol=1e-5)
    assert one["losses"][-1] != one["losses"][0]                                  # the solver moved (random data: no claim about the direction)


def test_iter_size_accumulation_equals_the_large_batch():
    """Solver::Step with iter_size = 2 on a batch of 32 (the same 32 samples twice) equals ... the gradient of those 32 samples:
    accumulate twice, scale by 1/iter_size (solver.cpp:277-288, sgd_solver.cpp Normalize)."""
    import multi_rank_worker as mw
    params, data, label = mw.build_case(32)
    a = mw.run(32, params, data, label, 3, iter_size=1)
    b = mw.run(32, params, data, label, 3, iter_size=2)
    for i in range(len(params)):
        assert rel(b[f"p{i}"], a[f"p{i}"]) < 1e-5, i

"""The reference's MNIST siamese example end to end through `tools/caffe.py train`, and the siamese-shaped net on two GPUs.

End to end: mnist_siamese_train_test.prototxt and mnist_siamese_solver.prototxt, unmodified but for the data sources (an LMDB of
synthetic 2x28x28 digit pairs instead of the LevelDB the example converts; sim = 1 when both halves come from the same synthetic
class), test_iter / test_interval (reduced so that periodic testing runs) and the snapshot prefix.  The loss falls; iteration 1's
logged loss is a float64 oracle's on the same first batch and initial weights; the TEST net's `loss` output is logged; the snapshot
loads into the deploy mnist_siamese.prototxt, whose `feat` equals the training net's on the same images."""
import os
import re
import socket
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from caffe_mpi_b200 import host_api, lmdb_io
import siamese_oracle as so

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SIAMESE = os.path.join(HERE, "golden", "reference_models", "examples", "siamese")
CLI = [sys.executable, os.path.join(ROOT, "tools", "caffe.py")]


def _digit(rng, cls):
    """one 28x28 uint8 image of synthetic class `cls` (0-9): a bright bar whose position and orientation the class fixes, jittered"""
    img = np.zeros((28, 28), np.uint8)
    r, c = 3 + 2 * (cls % 5) + rng.integers(0, 3), 4 + 2 * (cls // 5) * 5 + rng.integers(0, 3)
    if cls % 2:
        img[r:r + 12, c:c + 4] = rng.integers(160, 256)
    else:
        img[r:r + 4, c:c + 12] = rng.integers(160, 256)
    return img


def _pairs(rng, n):
    x = np.zeros((n, 2, 28, 28), np.uint8)
    sim = np.zeros(n, np.int64)
    for i in range(n):
        a = rng.integers(0, 10)
        b = a if rng.uniform() < 0.5 else rng.integers(0, 10)
        x[i, 0], x[i, 1] = _digit(rng, a), _digit(rng, b)
        sim[i] = int(a == b)
    return x, sim


def _setup(tmp_path):
    rng = np.random.default_rng(11)
    dbs = {}
    for split, n in (("train", 1280), ("test", 400)):
        x, sim = _pairs(rng, n)
        dbs[split] = str(tmp_path / ("siamese_%s_lmdb" % split))
        lmdb_io.write_datum_lmdb(dbs[split], x, sim)
    net = open(os.path.join(SIAMESE, "mnist_siamese_train_test.prototxt")).read()
    for split in ("train", "test"):
        src = 'source: "examples/siamese/mnist_siamese_%s_leveldb"' % split
        assert src in net
        net = net.replace(src, 'source: "%s"\n    backend: LMDB' % dbs[split])
    (tmp_path / "net.prototxt").write_text(net)
    solver = open(os.path.join(SIAMESE, "mnist_siamese_solver.prototxt")).read()
    solver = solver.replace('net: "examples/siamese/mnist_siamese_train_test.prototxt"', 'net: "%s"' % (tmp_path / "net.prototxt"))
    solver = solver.replace("test_iter: 100", "test_iter: 2").replace("test_interval: 500", "test_interval: 50")
    solver = solver.replace('snapshot_prefix: "examples/siamese/mnist_siamese"', 'snapshot_prefix: "%s"' % (tmp_path / "siam"))
    (tmp_path / "solver.prototxt").write_text(solver + "\nrandom_seed: 5\n")


def _tower(x, P):
    import torch.nn.functional as F
    h = F.max_pool2d(F.conv2d(x, P[0], P[1]), 2, 2)
    h = F.max_pool2d(F.conv2d(h, P[2], P[3]), 2, 2)
    h = F.relu(F.linear(h.reshape(h.shape[0], -1), P[4], P[5]))
    h = F.linear(h, P[6], P[7])
    return F.linear(h, P[8], P[9])


def test_reference_siamese_trains_end_to_end(tmp_path):
    _setup(tmp_path)
    r = subprocess.run(CLI + ["train", "--solver=solver.prototxt", "--iterations=200", "--display=50"], capture_output=True, text=True,
                       cwd=str(tmp_path), timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    losses = [float(x) for x in re.findall(r"Iteration \d+.*, loss = (\S+)", r.stdout)]
    assert len(losses) >= 4 and all(np.isfinite(losses)), r.stdout[-2000:]
    assert np.mean(losses[-2:]) < losses[0], losses
    # periodic testing ran at 0, 50, ... and logged the TEST net's ContrastiveLoss output
    text = r.stdout + r.stderr
    assert "Iteration 0, Testing net (#0)" in text and text.count("Testing net (#0)") >= 4, text[-2000:]
    test_losses = [float(x) for x in re.findall(r"Test net output #\d+: loss = (\S+)", text)]
    assert len(test_losses) >= 5 and all(np.isfinite(test_losses)), text[-2000:]
    model = str(tmp_path / "siam_iter_200.caffemodel")
    assert os.path.exists(model), os.listdir(tmp_path)

    # iteration 1's logged loss is the trainer's on the same net, solver and seed, and the float64 oracle's on its weights and batch
    r1 = subprocess.run(CLI + ["train", "--solver=solver.prototxt", "--iterations=1", "--display=1", "--snapshot_prefix=%s" % (tmp_path / "one")],
                        capture_output=True, text=True, cwd=str(tmp_path), timeout=900)
    assert r1.returncode == 0, r1.stderr[-3000:]
    logged = [float(x) for x in re.findall(r"Iteration 1 .*loss = (\S+)", r1.stdout)]
    assert len(logged) == 1, r1.stdout[-2000:]
    t = host_api.Trainer(str(tmp_path / "net.prototxt"), str(tmp_path / "solver.prototxt"), num_classes=2, seed=5, net_is_text=False,
                         solver_is_text=False)
    assert t.num_params() == 10
    first = t.forward_backward()
    assert first == pytest.approx(logged[0], rel=1e-5)
    pair = t.get_blob("pair_data").reshape(64, 2, 28, 28).astype(np.float64)
    sim = t.get_blob("sim").astype(np.float64)
    assert pair.max() <= 1.0 and pair.max() > 0.5                     # transform_param scale 1/256
    P = [torch.tensor(t.get_param(i, 0).astype(np.float64)).reshape(s) for i, s in
         enumerate([(20, 1, 5, 5), (20,), (50, 20, 5, 5), (50,), (500, 800), (500,), (10, 500), (10,), (2, 10), (2,)])]
    fa = _tower(torch.tensor(pair[:, 0:1]), P).numpy()
    fb = _tower(torch.tensor(pair[:, 1:2]), P).numpy()
    ref, _, _ = so.contrastive_forward(fa, fb, sim, margin=1.0)
    assert abs(first - ref) <= 1e-4 * abs(ref), (first, ref)

    # the snapshot in the deploy net: feat on the first halves equals the training net's feat on the same images
    t2 = host_api.Trainer(str(tmp_path / "net.prototxt"), str(tmp_path / "solver.prototxt"), num_classes=2, seed=5, net_is_text=False,
                          solver_is_text=False)
    assert t2.copy_trained_layers_from(model) > 0
    t2.forward_backward()
    imgs = t2.get_blob("pair_data").reshape(64, 2, 28, 28)
    feat = t2.get_blob("feat").reshape(64, 2)
    te = host_api.Tester(open(os.path.join(SIAMESE, "mnist_siamese.prototxt")).read(), batch=64, num_classes=2)
    te.copy_trained_layers_from(model)
    te.set_blob("data", np.ascontiguousarray(imgs[:, 0:1]))
    te.forward()
    np.testing.assert_allclose(te.get_blob("feat").reshape(64, 2), feat, rtol=1e-5, atol=1e-5 * float(np.abs(feat).max()))


def test_siamese_two_ranks_equal_one_rank():
    """Two processes, one GPU each (tests/siamese_rank_worker.py): the shared-weight net's parameters and momentum are bit-identical
    across ranks and equal one solver on the concatenated batch (1e-5 parameters, 1e-4 histories with a floor at 1e-3 of the
    largest), as tests/test_solvers_gpu.py's two-rank test states"""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import siamese_rank_worker as sw
    import test_siamese_sim as ss
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    global_batch, steps = 16, 3
    with tempfile.TemporaryDirectory() as td:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
               "--master-port", str(port), os.path.join(HERE, "siamese_rank_worker.py"), td, str(global_batch), str(steps)]
        r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-4000:])
        ranks = [dict(np.load(os.path.join(td, f"rank{i}.npz"))) for i in range(2)]
    params, data, label = ss.case(global_batch, seed=13)
    one = sw.run(global_batch, params, data, label, steps)
    for key in ("p", "h"):
        floor = 1e-20 if key == "p" else 1e-3 * max(float(np.abs(one[f"h{j}"]).max()) for j in range(len(params)))
        for i in range(len(params)):
            a, b = ranks[0][f"{key}{i}"], ranks[1][f"{key}{i}"]
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), f"{key}{i} differs across ranks"
            assert ss.rel(a, one[f"{key}{i}"], floor) < (1e-5 if key == "p" else 1e-4), (key, i)

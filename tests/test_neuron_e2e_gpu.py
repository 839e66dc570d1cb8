"""A conv + PReLU net end to end: `tools/caffe.py train` from an LMDB written with lmdb_io (the loss falls; iteration 1's logged loss
is the float64 oracle's on the same batch and initial weights), the snapshot scored by `caffe.py test` in the net's deploy form, and
the trained slopes -- per channel and channel-shared, the latter a 0-axis blob -- read back from the .caffemodel and giving the
oracle's `prob` in that deploy net.  With two GPUs, two ranks of the neuron net of tests/neuron_oracle.py end with bitwise-equal
slopes (tests/neuron_rank_worker.py)."""
import os
import re
import socket
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from caffe_mpi_b200 import host_api, lmdb_io
from test_snapshot_cpu import _schema

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CLI = [sys.executable, os.path.join(ROOT, "tools", "caffe.py")]
CLS, S, B = 4, 12, 16
SCALE = 0.00390625

LAYERS = (
    'layer { name: "conv1" type: "Convolution" bottom: "data" top: "conv1" convolution_param { num_output: 8 kernel_size: 3 pad: 1 '
    'weight_filler { type: "xavier" } } }\n'
    'layer { name: "pr1" type: "PReLU" bottom: "conv1" top: "conv1" }\n'
    'layer { name: "pool1" type: "Pooling" bottom: "conv1" top: "pool1" pooling_param { pool: MAX kernel_size: 2 stride: 2 } }\n'
    'layer { name: "conv2" type: "Convolution" bottom: "pool1" top: "conv2" convolution_param { num_output: 8 kernel_size: 3 pad: 1 '
    'weight_filler { type: "xavier" } } }\n'
    'layer { name: "pr2" type: "PReLU" bottom: "conv2" top: "p2" prelu_param { channel_shared: true } }\n'
    f'layer {{ name: "fc" type: "InnerProduct" bottom: "p2" top: "fc" inner_product_param {{ num_output: {CLS} '
    'weight_filler { type: "xavier" } } }\n')
# learnable ids: conv1 w, b; pr1 slope; conv2 w, b; pr2 slope (0-axis); fc w, b
SHAPES = [(8, 3, 3, 3), (8,), (8,), (8, 8, 3, 3), (8,), (), (CLS, 8 * (S // 2) ** 2), (CLS,)]
BLOBS = [("conv1", 2), ("pr1", 1), ("conv2", 2), ("pr2", 1), ("fc", 2)]


def _images(rng, n):
    """[n, 3, S, S] uint8: class k brightens quadrant k, with noise; labels uniform over the classes."""
    lab = rng.integers(0, CLS, n)
    img = rng.normal(90, 25, (n, 3, S, S))
    h = S // 2
    for i, k in enumerate(lab):
        img[i, :, (k // 2) * h:(k // 2 + 1) * h, (k % 2) * h:(k % 2 + 1) * h] += 110
    return np.clip(img, 0, 255).astype(np.uint8), lab


def forward(P, x, label=None):
    """float64: (loss or None, prob)"""
    import torch.nn.functional as F
    P = [torch.tensor(np.asarray(p, np.float64)) for p in P]
    X = torch.tensor(np.asarray(x, np.float64))
    c1 = F.conv2d(X, P[0].reshape(SHAPES[0]), P[1], padding=1)
    c1 = torch.where(c1 > 0, c1, c1 * P[2].reshape(1, -1, 1, 1))
    p1 = F.max_pool2d(c1, 2, 2)
    c2 = F.conv2d(p1, P[3].reshape(SHAPES[3]), P[4], padding=1)
    p2 = torch.where(c2 > 0, c2, c2 * P[5].reshape(-1))
    fc = p2.reshape(p2.shape[0], -1) @ P[6].reshape(SHAPES[6]).T + P[7]
    loss = None if label is None else float(F.cross_entropy(fc, torch.tensor(np.asarray(label).astype(np.int64))))
    return loss, torch.softmax(fc, 1).numpy()


def _setup(tmp_path):
    rng = np.random.default_rng(23)
    src = {}
    for split, n in (("train", 256), ("test", 64)):
        src[split] = str(tmp_path / ("prelu_%s_lmdb" % split))
        lmdb_io.write_datum_lmdb(src[split], *_images(rng, n))
    data = ''
    for phase in ("TRAIN", "TEST"):
        data += (f'layer {{ name: "data" type: "Data" top: "data" top: "label" include {{ phase: {phase} }}\n'
                 f'  transform_param {{ scale: {SCALE} }} data_param {{ source: "{src[phase.lower()]}" backend: LMDB batch_size: {B} }} }}\n')
    tail = ('layer { name: "loss" type: "SoftmaxWithLoss" bottom: "fc" bottom: "label" top: "loss" }\n'
            'layer { name: "acc" type: "Accuracy" bottom: "fc" bottom: "label" top: "acc" include { phase: TEST } }\n')
    (tmp_path / "net.prototxt").write_text('name: "prelu"\n' + data + LAYERS + tail)
    deploy = (f'name: "prelu"\nlayer {{ name: "data" type: "Input" top: "data" input_param {{ shape {{ dim: {B} dim: 3 dim: {S} dim: {S} }} }} }}\n'
              + LAYERS + 'layer { name: "prob" type: "Softmax" bottom: "fc" top: "prob" }\n')
    (tmp_path / "deploy.prototxt").write_text(deploy)
    (tmp_path / "solver.prototxt").write_text(
        f'net: "{tmp_path / "net.prototxt"}"\ntest_iter: 2\ntest_interval: 40\nbase_lr: 0.02\nmomentum: 0.9\nlr_policy: "fixed"\n'
        f'display: 1\nmax_iter: 80\nsnapshot_prefix: "{tmp_path / "prelu"}"\nrandom_seed: 5\n')
    return deploy


def _caffemodel_blobs(path):
    """{layer: [(shape, float32 data)]} of a .caffemodel, parsed by google.protobuf"""
    m = _schema()["NetParameter"]()
    with open(path, "rb") as f:
        m.ParseFromString(f.read())
    out = {}
    for layer in m.layer:
        bl = []
        for b in layer.blobs:
            data = np.frombuffer(b.raw_data, np.float32).copy() if b.HasField("raw_data") else np.array(b.data, np.float32)
            bl.append((tuple(b.shape.dim), data))
        out[layer.name] = bl
    return out


def test_prelu_net_trains_and_scores_end_to_end(tmp_path):
    deploy = _setup(tmp_path)
    r = subprocess.run(CLI + ["train", "--solver=solver.prototxt", "--iterations=80", "--display=1"], capture_output=True, text=True,
                       cwd=str(tmp_path), timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    losses = [float(x) for x in re.findall(r"Iteration \d+.*, loss = (\S+)", r.stdout)]
    assert len(losses) == 80 and all(np.isfinite(losses)), r.stdout[-2000:]
    assert np.mean(losses[-10:]) < 0.5 * losses[0], losses
    model = str(tmp_path / "prelu_iter_80.caffemodel")
    assert os.path.exists(model), os.listdir(tmp_path)

    # iteration 1's logged loss is the trainer's on the same net, solver and seed, and the float64 oracle's on its batch and weights
    r1 = subprocess.run(CLI + ["train", "--solver=solver.prototxt", "--iterations=1", "--display=1", "--snapshot_prefix=%s" % (tmp_path / "one")],
                        capture_output=True, text=True, cwd=str(tmp_path), timeout=900)
    assert r1.returncode == 0, r1.stderr[-3000:]
    logged = [float(x) for x in re.findall(r"Iteration 1 .*loss = (\S+)", r1.stdout)]
    assert len(logged) == 1, r1.stdout[-2000:]
    t = host_api.Trainer(str(tmp_path / "net.prototxt"), str(tmp_path / "solver.prototxt"), num_classes=CLS, seed=5, net_is_text=False,
                         solver_is_text=False)
    assert t.num_params() == len(SHAPES)
    np.testing.assert_array_equal(t.get_param(2, 0), np.full(8, 0.25, np.float32))      # the default filler, both slope forms
    np.testing.assert_array_equal(t.get_param(5, 0), np.full(1, 0.25, np.float32))
    first = t.forward_backward()
    assert first == pytest.approx(logged[0], rel=1e-5)
    data = t.get_blob("data").reshape(B, 3, S, S)
    label = t.get_blob("label")
    assert data.max() <= 1.0 and data.max() > 0.5                                     # transform_param scale 1/256
    ref, _ = forward([t.get_param(i, 0) for i in range(len(SHAPES))], data, label)
    assert abs(first - ref) <= 1e-4 * abs(ref), (first, ref)

    # the snapshot: slopes trained away from the filler, the shared one a 0-axis blob; scored by caffe.py test in the deploy form
    blobs = _caffemodel_blobs(model)
    (s1_shape, s1), = blobs["pr1"]
    (s2_shape, s2), = blobs["pr2"]
    assert s1_shape == (8,) and s2_shape == ()
    assert s2.size == 1 and s2[0] != 0.25 and np.any(s1 != 0.25)
    r2 = subprocess.run(CLI + ["test", "--model=deploy.prototxt", "--weights=%s" % model, "--iterations=1"], capture_output=True,
                        text=True, cwd=str(tmp_path), timeout=900)
    assert r2.returncode == 0, r2.stderr[-3000:]
    probs = [float(v) for v in re.findall(r"Batch 0, prob = (\S+)", r2.stdout + r2.stderr)]
    assert len(probs) == B * CLS and all(0.0 <= p <= 1.0 for p in probs), (r2.stdout + r2.stderr)[-3000:]
    # ... and the slopes round-trip: the deploy net on those weights gives the oracle's prob on the same images
    P = [arr for name, n in BLOBS for _, arr in blobs[name][:n]]
    te = host_api.Tester(deploy, batch=B, num_classes=CLS)
    te.copy_trained_layers_from(model)
    te.set_blob("data", data)
    te.forward()
    _, want = forward(P, data)
    np.testing.assert_allclose(te.get_blob("prob").reshape(B, CLS), want, rtol=1e-4, atol=1e-5)


def test_two_ranks_end_with_bitwise_equal_slopes():
    """Two processes, one GPU each (tests/neuron_rank_worker.py): every parameter, the slopes of both forms included, is bit-identical
    across ranks after three SGD steps, and equals one solver on the concatenated batch"""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import neuron_rank_worker as nw
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    global_batch, steps = 8, 3
    for shared in (0, 1):
        with tempfile.TemporaryDirectory() as td:
            cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                   "--master-port", str(port + shared), os.path.join(HERE, "neuron_rank_worker.py"), td, str(global_batch), str(steps),
                   str(shared)]
            r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
            assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-4000:])
            ranks = [dict(np.load(os.path.join(td, f"rank{i}.npz"))) for i in range(2)]
        params, data, label = nw.case(global_batch, bool(shared))
        one = nw.run(global_batch, params, data, label, steps, bool(shared))
        for i in range(len(params)):
            a, b = ranks[0][f"p{i}"], ranks[1][f"p{i}"]
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), f"parameter {i} differs across ranks"
            assert float(np.abs(a - one[f"p{i}"]).max()) <= 1e-5 * max(float(np.abs(one[f"p{i}"]).max()), 1e-6), i

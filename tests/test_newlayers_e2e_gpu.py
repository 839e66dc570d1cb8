"""The reference's own model files that use Softmax / Sigmoid / Flatten / SigmoidCrossEntropyLoss / EuclideanLoss, end to end through
`tools/caffe.py train`: the MNIST autoencoder on a 1x28x28 LMDB (the loss falls; its first value is the net oracle's on the same
first batch and initial weights), and Inception-v2 with periodic testing (its TEST net's Softmax -> Accuracy outputs are logged)."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from caffe_mpi_b200 import host_api, lmdb_io
import newlayers_oracle as nlo

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.path.join(HERE, "golden", "reference_models")
CLI = [sys.executable, os.path.join(ROOT, "tools", "caffe.py")]


def _lines(out):
    return [ln.split("caffe.py] ", 1)[1] for ln in out.splitlines() if "caffe.py] " in ln]


def _digits(rng, n):
    """MNIST-like uint8 images: black, with a bright stroke (a random rectangle) each."""
    img = np.zeros((n, 1, 28, 28), np.uint8)
    for i in range(n):
        r, c = rng.integers(2, 16, 2)
        h, w = rng.integers(4, 12, 2)
        img[i, 0, r:r + h, c:c + w] = rng.integers(128, 256)
    return img


def test_reference_autoencoder_trains_from_lmdb(tmp_path, monkeypatch):
    monkeypatch.delenv("B2C_DATA", raising=False)
    rng = np.random.default_rng(3)
    db = str(tmp_path / "mnist_train_lmdb")
    lmdb_io.write_datum_lmdb(db, _digits(rng, 1000), rng.integers(0, 10, 1000))
    net = open(os.path.join(REF, "examples/mnist/mnist_autoencoder.prototxt")).read().replace("examples/mnist/mnist_train_lmdb", db)
    (tmp_path / "net.prototxt").write_text(net)
    # mnist_autoencoder_solver_nesterov.prototxt without its test_* lines (test_state stages are not built), run for 300 iterations
    solver = [ln for ln in open(os.path.join(REF, "examples/mnist/mnist_autoencoder_solver_nesterov.prototxt")).read().splitlines()
              if not ln.startswith("test_") and not ln.startswith("net:") and not ln.startswith("snapshot")]
    (tmp_path / "solver.prototxt").write_text('net: "%s"\n' % (tmp_path / "net.prototxt") + "\n".join(solver) + "\nrandom_seed: 5\n")
    r = subprocess.run(CLI + ["train", "--solver=solver.prototxt", "--iterations=300", "--display=50"], capture_output=True, text=True,
                       cwd=str(tmp_path), timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    assert "with Nesterov:" in r.stdout
    losses = [float(x) for x in re.findall(r"loss = (\S+)", r.stdout)]
    assert len(losses) >= 6 and all(np.isfinite(losses)), r.stdout[-2000:]
    assert all(b < a for a, b in zip(losses, losses[1:])) and losses[-1] < 0.7 * losses[0], losses
    # iteration 1's loss line (the first step's forward, on the initial weights and the first batch) ...
    r1 = subprocess.run(CLI + ["train", "--solver=solver.prototxt", "--iterations=1", "--display=1"], capture_output=True, text=True,
                        cwd=str(tmp_path), timeout=900)
    assert r1.returncode == 0, r1.stderr[-3000:]
    logged = [float(x) for x in re.findall(r"Iteration 1 .*loss = (\S+)", r1.stdout)]
    assert len(logged) == 1, r1.stdout[-2000:]
    # ... is the trainer API's on the same net, solver and seed, and the net oracle's on its weights and first batch
    t = host_api.Trainer(str(tmp_path / "net.prototxt"), str(tmp_path / "solver.prototxt"), num_classes=10, seed=5, net_is_text=False,
                         solver_is_text=False)
    first = t.forward_backward()
    assert first == pytest.approx(logged[0], rel=1e-5)                  # (the log prints six significant digits)
    assert losses[0] < first
    spec = nlo.autoencoder(batch=100, side=28, widths=(1000, 500, 250, 30))
    params = [t.get_param(i, 0).reshape(shp) for i, (_, _, shp) in enumerate(nlo.param_shapes(spec))]
    data = t.get_blob("data").reshape(100, 1, 28, 28)
    assert data.max() <= 1.0 and data.max() > 0.4                   # transform_param scale 1/255 applied
    ref_loss, grads, _ = nlo.forward_backward(spec, params, data)
    assert abs(first - ref_loss) <= 1e-4 * abs(ref_loss), (first, ref_loss)
    assert t.get_blob("cross_entropy_loss")[0] == pytest.approx(first, rel=0)
    # gradients at the north-star bar (DESIGN section 4): the reference's std-1 gaussian filler (its `sparse: 15` is not read) puts
    # encode1's pre-activations at a standard deviation near 16, so the sigmoids sit in saturation, where y (1 - y) keeps few digits
    # of float32, and the deepest blob's gradient passes eight InnerProduct layers and seven of those derivatives (about 8e-4 there)
    errs = [float(np.abs(t.get_param(i, 1).reshape(-1) - g.reshape(-1)).max()) / max(float(np.abs(g).max()), 1e-20) for i, g in enumerate(grads)]
    assert max(errs) <= 1e-3, errs
    assert max(errs[-2:]) <= 1e-4, errs                                 # decode1, the InnerProduct next to the loss: the 1e-4 bar


def test_reference_inception_v2_trains_with_periodic_testing(tmp_path):
    text = open(os.path.join(REF, "models/inception_v2/solver.prototxt")).read()
    text = text.replace("test_iter: 1562", "test_iter: 2").replace("test_interval: 20000", "test_interval: 2")
    (tmp_path / "solver.prototxt").write_text(text)
    r = subprocess.run(CLI + ["train", "--solver=%s" % (tmp_path / "solver.prototxt"), "--iterations=2", "--batch=8", "--display=1",
                              "--snapshot_prefix=%s" % (tmp_path / "s")],
                       capture_output=True, text=True, cwd=REF, timeout=900, env=dict(os.environ, B2C_DATA="synthetic"))
    assert r.returncode == 0, r.stderr[-3000:]
    losses = [float(x) for x in re.findall(r"loss = (\S+)", r.stdout)]
    assert len(losses) == 2 and all(np.isfinite(losses))
    lines = _lines(r.stderr)
    assert "Iteration 0, Testing net (#0)" in lines and "Iteration 2, Testing net (#0)" in lines
    outs = [re.match(r"\s*Test net output #\d+: (\S+) = (\S+)", ln) for ln in lines]
    scores = {}
    for mt in outs:
        if mt:
            scores.setdefault(mt.group(1), []).append(float(mt.group(2)))
    # the auxiliary classifiers' Softmax -> Accuracy outputs, and the main classifier's
    for k in ("loss1/top-1", "loss1/top-5", "loss2/top-1", "loss2/top-5", "accuracy/top-1", "accuracy/top-5"):
        assert k in scores and len(scores[k]) == 2, (k, sorted(scores))
        assert all(0.0 <= v <= 1.0 for v in scores[k])
    assert all(np.isfinite(v).all() for v in map(np.array, scores.values()))

"""Periodic testing inside `caffe.py train` on the GPU: the logged test scores against the Tester on the matching snapshots, training
untouched by the passes, the test pass against Tester.test bit for bit, two ranks against one GPU, the reference ResNet-50 solver, and
the reference's solver files (which all carry test nets) through the shell."""
import importlib.util
import os
import re
import socket
import subprocess
import sys

import numpy as np
import pytest

from caffe_mpi_b200 import host_api, lmdb_io
import netoracle as no

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.path.join(HERE, "golden", "reference_models")
CLI = [sys.executable, os.path.join(ROOT, "tools", "caffe.py")]
_spec = importlib.util.spec_from_file_location("caffe_cli_periodic_gpu", CLI[1])
cli = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(cli)


def _line_text(out):
    return [ln.split("caffe.py] ", 1)[1] for ln in out.splitlines() if "caffe.py] " in ln]


def _mini_resnet_net(train, test, batch, test_batch):
    body = [ln for ln in no.to_prototxt(no.mini_resnet(batch=batch)).splitlines() if 'type: "Input"' not in ln and not ln.startswith("name:")]
    data = "".join(f'layer {{ name: "data" type: "Data" top: "data" top: "label" include {{ phase: {ph} }} transform_param {{ scale: 0.0078125 }}\n'
                   f'  data_param {{ source: "{src}" batch_size: {b} backend: LMDB }} }}\n'
                   for ph, src, b in (("TRAIN", train, batch), ("TEST", test, test_batch)))
    acc = 'layer { name: "accuracy" type: "Accuracy" bottom: "fc" bottom: "label" top: "accuracy" include { phase: TEST } }\n'
    return 'name: "mini"\n' + data + "\n".join(body) + "\n" + acc


def _databases(tmp_path, rng, shape=(3, 16, 16), n_train=64, n_test=48):
    out = []
    for name, n in (("train_lmdb", n_train), ("val_lmdb", n_test)):
        path = str(tmp_path / name)
        lmdb_io.write_datum_lmdb(path, rng.integers(0, 256, (n,) + shape, dtype=np.uint8), rng.integers(0, 10, n))
        out.append(path)
    return out


SOLVER = 'base_lr: 0.05 lr_policy: "fixed" momentum: 0.9 weight_decay: 0.0005 solver_mode: GPU random_seed: 5 snapshot_prefix: "snap"\n'


def test_logged_scores_are_the_testers_on_the_snapshots_and_training_is_untouched(tmp_path, monkeypatch):
    monkeypatch.delenv("B2C_DATA", raising=False)
    rng = np.random.default_rng(21)
    train, val = _databases(tmp_path, rng)
    net = tmp_path / "train_val.prototxt"
    net.write_text(_mini_resnet_net(train, val, 4, 4))
    runs = {}
    for tag, extra in (("tested", "test_iter: 3 test_interval: 2\n"), ("plain", "")):
        d = tmp_path / tag
        d.mkdir()
        (d / "solver.prototxt").write_text(f'net: "{net}"\n' + SOLVER + "max_iter: 6 snapshot: 2\n" + extra)
        # stdout (training) and stderr (test nets) as one stream, in the order they were written
        r = subprocess.run(CLI + ["train", "--solver=solver.prototxt", "--classes=10"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                           cwd=str(d), timeout=600)
        assert r.returncode == 0, r.stdout[-3000:]
        runs[tag] = (d, _line_text(r.stdout))
    d, lines = runs["tested"]
    assert not any("Testing net" in ln for ln in runs["plain"][1])
    # the final weights, BatchNorm statistics and momentum do not see the passes
    for ext in (".caffemodel", ".solverstate"):
        assert (d / ("snap_iter_6" + ext)).read_bytes() == (runs["plain"][0] / ("snap_iter_6" + ext)).read_bytes(), ext
    # the passes: at 0 (one batch), at 2 and 4 (before those iterations, after their snapshots) and after the last iteration
    heads = [i for i, ln in enumerate(lines) if re.match(r"Iteration \d+, Testing net \(#0\)", ln)]
    assert [lines[i] for i in heads] == ["Iteration %d, Testing net (#0)" % k for k in (0, 2, 4, 6)]
    assert "Initial Test completed" in lines and sum(ln.startswith("Tests completed in ") for ln in lines) == 2
    snaps = [i for i, ln in enumerate(lines) if ln.startswith("Snapshotting")]
    assert snaps[0] < heads[1] < snaps[1] < heads[2] < snaps[2] < heads[3]
    trainer = host_api.Trainer(str(net), str(d / "solver.prototxt"), num_classes=10, seed=5, net_is_text=False, solver_is_text=False)
    consumed = 0
    for k, it in enumerate((0, 2, 4, 6)):
        te = host_api.Tester(str(net), num_classes=10, seed=5, net_is_text=False)
        if it == 0:
            te.share_trained_layers_with(trainer)                             # the weights training starts from
        else:
            te.copy_trained_layers_from(str(d / ("snap_iter_%d.caffemodel" % it)))
        for _ in range(consumed):                                             # the shell's reader is never rewound
            te.forward()
        batches = 1 if it == 0 else 3
        means, loss = te.test_pass(batches)
        consumed += batches
        logged = [ln.strip() for ln in lines[heads[k] + 1:heads[k] + 3]]
        assert logged == [ln.strip() for ln in cli.test_net_lines(te.outputs(), means, loss, False)], (it, logged)


def test_test_pass_is_test_bit_for_bit_on_one_gpu(tmp_path, monkeypatch):
    monkeypatch.delenv("B2C_DATA", raising=False)
    rng = np.random.default_rng(22)
    train, val = _databases(tmp_path, rng)
    net = _mini_resnet_net(train, val, 4, 4)
    t = host_api.Trainer(net, SOLVER, num_classes=10)
    t.step(3, copy_input=True)
    a, b = host_api.Tester(net, num_classes=10), host_api.Tester(net, num_classes=10)
    a.share_trained_layers_with(t)
    b.share_trained_layers_with(t)
    for k in (1, 5):
        _, means, _ = a.test(k)
        got, _ = b.test_pass(k)
        assert np.array_equal(got.view(np.uint32), means.view(np.uint32)), k
        t.step(2, copy_input=True)


def _scores(lines):
    return [float(m.group(1)) for m in (re.match(r"\s*Test net output #\d+: \S+ = (\S+)", ln) for ln in lines) if m]


def test_two_ranks_score_what_one_gpu_scores_on_the_whole_batch(tmp_path, monkeypatch):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    monkeypatch.delenv("B2C_DATA", raising=False)
    rng = np.random.default_rng(23)
    train, val = _databases(tmp_path, rng, shape=(3, 8, 8))
    net = tmp_path / "net.prototxt"
    net.write_text('name: "ipnet"\n'
                   f'layer {{ name: "data" type: "Data" top: "data" top: "label" include {{ phase: TRAIN }} transform_param {{ scale: 0.0078125 }} data_param {{ source: "{train}" batch_size: 8 backend: LMDB }} }}\n'
                   f'layer {{ name: "data" type: "Data" top: "data" top: "label" include {{ phase: TEST }} transform_param {{ scale: 0.0078125 }} data_param {{ source: "{val}" batch_size: 8 backend: LMDB }} }}\n'
                   'layer { name: "ip" type: "InnerProduct" bottom: "data" top: "ip" inner_product_param { num_output: 10 weight_filler { type: "gaussian" std: 0.1 } } }\n'
                   'layer { name: "loss" type: "SoftmaxWithLoss" bottom: "ip" bottom: "label" top: "loss" }\n'
                   'layer { name: "accuracy" type: "Accuracy" bottom: "ip" bottom: "label" top: "accuracy" include { phase: TEST } }\n')
    solver = tmp_path / "solver.prototxt"          # base_lr 0: both runs score the same weights at every pass
    solver.write_text(f'net: "{net}"\nbase_lr: 0 lr_policy: "fixed" max_iter: 4 test_iter: 2 test_interval: 2 random_seed: 5 solver_mode: GPU\n')
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    two = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                          "--master-port", str(port), os.path.join(ROOT, "tools", "caffe.py"), "train", "--solver=%s" % solver, "--classes=10"],
                         capture_output=True, text=True, cwd=ROOT, timeout=600)
    assert two.returncode == 0, two.stderr[-3000:]
    one = subprocess.run(CLI + ["train", "--solver=%s" % solver, "--classes=10"], capture_output=True, text=True, cwd=ROOT, timeout=600)
    assert one.returncode == 0, one.stderr[-3000:]
    a, b = _scores(_line_text(two.stderr)), _scores(_line_text(one.stderr))
    assert len(a) == len(b) == 6 and "[MultiGPU] Initial Test completed" in two.stderr
    np.testing.assert_allclose(a, b, rtol=0, atol=1e-6)


def test_reference_resnet50_solver_tests_on_the_synthetic_source(tmp_path):
    text = open(os.path.join(REF, "models", "resnet50", "solver.prototxt")).read().replace("test_iter: 1562", "test_iter: 2")
    solver = tmp_path / "solver.prototxt"
    solver.write_text(text)
    r = subprocess.run(CLI + ["train", "--solver=%s" % solver, "--iterations=4", "--display=1", "--snapshot_prefix=%s" % (tmp_path / "s")],
                       capture_output=True, text=True, cwd=REF, timeout=900, env=dict(os.environ, B2C_DATA="synthetic"))
    assert r.returncode == 0, r.stderr[-3000:]
    lines = _line_text(r.stderr)
    assert "Iteration 0, Testing net (#0)" in lines and "Initial Test completed" in lines
    outs = [re.match(r"\s*Test net output #\d+: (\S+) = (\S+)", ln) for ln in lines]
    scores = {m.group(1): float(m.group(2)) for m in outs if m}
    assert set(scores) == {"accuracy/top-1", "accuracy/top-5", "loss"} and all(np.isfinite(list(scores.values())))
    assert all(0.0 <= v <= 1.0 for k, v in scores.items() if k.startswith("accuracy"))


@pytest.mark.parametrize("solver,classes", [("examples/solvers/adam/solver.prototxt", 1000),
                                            ("examples/mnist/lenet_solver_rmsprop.prototxt", 10)])
def test_reference_solver_files_log_their_test_passes_on_stderr(solver, classes, tmp_path):
    """The reference's solver files carry test nets: the one-batch pass at iteration 0 is logged on stderr, and stdout holds the same
    lines as without test nets -- three training losses for three iterations, no test line.  No pass runs at the iteration a resumed
    run starts from."""
    env = dict(os.environ, B2C_DATA="synthetic")
    prefix = str(tmp_path / "snap")
    base = CLI + ["train", "--solver=" + solver, "--batch=64", "--display=1", "--classes=%d" % classes]
    r = subprocess.run(base + ["--iterations=3", "--snapshot_prefix=" + prefix], capture_output=True, text=True, cwd=REF, timeout=600, env=env)
    assert r.returncode == 0, r.stderr[-3000:]
    losses = [float(x) for x in re.findall(r"loss = (\S+)", r.stdout)]
    assert len(losses) == 3 and all(np.isfinite(losses)) and "Test" not in r.stdout, r.stdout
    lines = _line_text(r.stderr)
    assert lines[1:2] == ["Iteration 0, Testing net (#0)"] and "Initial Test completed" in lines and lines[0].startswith("Creating test net (#0)")
    assert _scores(lines) and all(np.isfinite(_scores(lines)))
    r2 = subprocess.run(base + ["--iterations=2", "--snapshot=" + prefix + "_iter_3.solverstate", "--snapshot_prefix=" + prefix], capture_output=True, text=True, cwd=REF,
                        timeout=600, env=env)
    assert r2.returncode == 0, r2.stderr[-3000:]
    assert "Iteration 5 (" in r2.stdout and "Testing net" not in r2.stderr

"""The TEST phase without a GPU: the oracle's inference BatchNorm against a hand-computed vector, the five BASELINE nets built as TEST
nets from the stored reference prototxts, weight sharing / copying refusing shape mismatches, the TEST forward of the mini nets on
the host stand-ins of tests/sim (libinfersim.so) against tests/infer_oracle.py, and the `caffe.py test` shell."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from caffe_mpi_b200 import capi, host_api
import infer_oracle as io_
import netoracle as no

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.path.join(HERE, "golden", "reference_models")
SOLVER = 'base_lr: 0.05 lr_policy: "fixed" momentum: 0.9 weight_decay: 0.0005 max_iter: 100 solver_mode: GPU'
ACCURACY = 'layer { name: "accuracy" type: "Accuracy" bottom: "fc" bottom: "label" top: "accuracy" }\n'


def test_oracle_bn_inference_known_answer_with_double_eps():
    # running_var = 3.875 already holds variance + eps (eps = 0.125 added on the TRAIN side); TEST adds eps again: 1/sqrt(4) = 0.5.
    # A single eps would give 1/sqrt(3.875).
    x = np.array([1, 3, 5, -7, 2, 2, 2, 2], np.float32).reshape(2, 1, 2, 2).transpose(1, 0, 2, 3).copy()   # N = 1, C = 2, S = 4
    mean, var = np.array([1, 2], np.float32), np.array([3.875, 0.875], np.float32)
    gamma, beta = np.array([2, 4], np.float32), np.array([0.5, -1], np.float32)
    y = io_.bn_forward_inference(x, gamma, beta, 0.125, mean, var)
    np.testing.assert_array_equal(y.reshape(-1), [0.5, 2.5, 4.5, -7.5, -1, -1, -1, -1])
    y = io_.bn_forward_inference(x, None, None, 0.125, mean, var, residual=np.full_like(x, -1), relu=True)
    np.testing.assert_array_equal(y.reshape(-1), [0, 0, 1, 0, 0, 0, 0, 0])


@pytest.fixture(scope="module")
def sim_host():
    """host_api pointed at libinfersim.so (tests/sim: the host layer over stand-in kernels, the TEST-phase BatchNorm included) for the
    duration of the module."""
    capi.lib()
    r = subprocess.run(["make", "-C", os.path.join(HERE, "sim"), "-f", "Makefile.infer", "libinfersim.so"], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.fail("tests/sim/libinfersim.so does not build:\n" + r.stdout[-1000:] + r.stderr[-3000:])
    saved = (host_api._lib, host_api._SO, os.environ.get("B2C_NCCL_ARENA"))
    host_api._lib, host_api._SO = None, os.path.join(HERE, "sim", "libinfersim.so")
    os.environ["B2C_NCCL_ARENA"] = "0"
    try:
        L = host_api.lib()
        L.fakecuda_set_all_eager.argtypes = [C.c_int]
        L.fakecuda_set_all_eager(0)
        yield host_api
    finally:
        host_api._lib, host_api._SO = saved[0], saved[1]
        if saved[2] is None:
            os.environ.pop("B2C_NCCL_ARENA", None)
        else:
            os.environ["B2C_NCCL_ARENA"] = saved[2]


TOP = [("accuracy/top-1", 0.0), ("accuracy/top-5", 0.0), ("loss", 1.0)]
NETS = {
    "resnet50": ("models/resnet50/train_val.prototxt", 32, TOP),
    "alexnet": ("models/bvlc_alexnet/train_val.prototxt", 32, TOP),
    "vgg16": ("models/vgg16/train_val.prototxt", 32, TOP),
    # the three heads at 0.3 / 0.3 / 1 (the auxiliary losses' tops are loss1/loss1 and loss2/loss1 in the reference's file)
    "googlenet": ("models/bvlc_googlenet/train_val.prototxt", 32,
                  TOP + [(f"loss{k}/{t}", 0.3 if t == "loss1" else 0.0) for k in "12" for t in ("loss1", "top-1", "top-5")]),
    "lenet": ("examples/mnist/lenet_train_test.prototxt", 100, [("accuracy", 0.0), ("loss", 1.0)]),
}


@pytest.mark.parametrize("name", sorted(NETS))
def test_reference_nets_build_as_test_nets(sim_host, name):
    path, batch, outputs = NETS[name]
    path = os.path.join(REF, path)
    kw = dict(default_channels=1, default_size=28) if name == "lenet" else {}
    data = [l for l in sim_host.Net(path, phase="TEST", **kw).layers() if l[1] == "Data"]
    assert len(data) == 1 and data[0][2][0] == batch                    # the TEST data layer's own batch_size
    t = sim_host.Tester(path, batch=2, num_classes=10 if name == "lenet" else 1000, net_is_text=False, **kw)
    got = t.outputs()
    assert [(n, round(w, 6)) for n, w, _ in got] == outputs                        # Net::output_blobs in name order, with loss weights
    assert all(c == 1 for _, _, c in got)
    assert not t.has_solver()                                            # forward only: no SGDSolver, no parameter arena
    assert [ty for _, ty in t.layers()].count("Data") == 1


def test_share_and_copy_refuse_a_shape_mismatch(sim_host, tmp_path):
    spec10, spec7 = no.mini_resnet(classes=10), no.mini_resnet(classes=7)
    tr = sim_host.Trainer(no.to_prototxt(spec10), SOLVER, num_classes=10)
    te = sim_host.Tester(no.to_prototxt(spec7), num_classes=7)
    with pytest.raises(host_api.HostError, match="layer 'fc'; shape mismatch"):
        te.share_trained_layers_with(tr)
    model = tr.snapshot(str(tmp_path / "m")).replace(".solverstate", ".caffemodel")
    with pytest.raises(host_api.HostError, match="from layer 'fc'; shape mismatch"):
        te.copy_trained_layers_from(model)
    ok = sim_host.Tester(no.to_prototxt(spec10), num_classes=10)
    ok.share_trained_layers_with(tr)
    assert ok.copy_trained_layers_from(model) == len(io_.model_layers(spec10, *io_.random_model(spec10, np.random.default_rng(0))))


def _check_test_forward(host, spec, rng, tmp_path, names):
    params, stats = io_.random_model(spec, rng)
    path = str(tmp_path / "w.caffemodel")
    io_.write_caffemodel(host.lib(), path, io_.model_layers(spec, params, stats))
    t = host.Tester(no.to_prototxt(spec) + ACCURACY.replace('"fc"', '"%s"' % spec[-1]["b"][0]), num_classes=10)
    assert t.copy_trained_layers_from(path) == len(io_.model_layers(spec, params, stats))
    data = rng.standard_normal(spec[0]["shape"]).astype(np.float32)
    label = rng.integers(0, 10, spec[0]["shape"][0]).astype(np.float32)
    t.set_blob("data", data)
    t.set_blob("label", label)
    t.forward()
    v = io_.forward_test_phase(spec, params, stats, data, label)
    for n in names:
        ref = v[n]
        assert np.max(np.abs(t.get_blob(n) - ref.reshape(-1))) <= 1e-4 * max(np.max(np.abs(ref)), 1e-20), n
    from oracle import layers_oracle as lo
    acc = lo.accuracy(v[spec[-1]["b"][0]], label)
    per_batch, means, loss = t.test(2)
    outs = t.outputs()
    ref_loss = sum(w * float(v[n]) for n, w, _ in outs if w)
    assert abs(loss - ref_loss) <= 1e-4 * abs(ref_loss)
    for k, (n, w, _) in enumerate(outs):
        ref = float(acc) if n == "accuracy" else float(v[n])
        assert abs(means[k] - ref) <= 1e-4 * max(abs(ref), 1e-6) and abs(per_batch[1][k] - ref) <= 1e-4 * max(abs(ref), 1e-6), n
    return t, outs


def test_mini_resnet_test_forward_matches_the_oracle_on_the_cpu(sim_host, rng, tmp_path):
    spec = no.mini_resnet()
    _, outs = _check_test_forward(sim_host, spec, rng, tmp_path, ["conv1", "pool1", "resA.1.sum", "resA.2.sum", "pool2", "fc"])
    assert [(n, w) for n, w, _ in outs] == [("accuracy", 0.0), ("loss", 1.0)]


def test_mini_inception_test_forward_matches_the_oracle_on_the_cpu(sim_host, rng, tmp_path):
    spec = no.mini_inception()
    _, outs = _check_test_forward(sim_host, spec, rng, tmp_path, ["conv1", "norm1", "inc/output", "aux/fc", "pool5", "cls"])
    assert [(n, round(w, 6)) for n, w, _ in outs] == [("accuracy", 0.0), ("aux/loss1", 0.3), ("loss", 1.0)]


def _caffe(*args):
    return subprocess.run([sys.executable, os.path.join(ROOT, "tools", "caffe.py"), *args], capture_output=True, text=True, cwd=ROOT)


def test_caffe_test_argument_errors():
    r = _caffe("test", "--weights=x.caffemodel")
    assert r.returncode != 0 and "Need a model definition to score." in r.stderr
    r = _caffe("test", "--model=x.prototxt")
    assert r.returncode != 0 and "Need model weights to score." in r.stderr


def test_caffe_test_score_lines_follow_the_reference_layout():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import caffe as cli
    outputs = [("accuracy", 0.0, 1), ("loss", 1.0, 1), ("loss1/loss1", 0.3, 1)]
    lines = cli.score_lines(outputs, [[0.5, 2.25, 3.0], [0.25, 1.75, 2.0]], [0.375, 2.0, 2.5], 2.75)
    assert lines == ["Batch 0, accuracy = 0.5", "Batch 0, loss = 2.25", "Batch 0, loss1/loss1 = 3",
                     "Batch 1, accuracy = 0.25", "Batch 1, loss = 1.75", "Batch 1, loss1/loss1 = 2",
                     "Loss: 2.75",
                     "accuracy = 0.375", "loss = 2 (* 1 = 2 loss)", "loss1/loss1 = 2.5 (* 0.3 = 0.75 loss)"]

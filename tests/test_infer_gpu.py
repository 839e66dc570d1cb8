"""The TEST phase on the device: b2c_bn_forward_inference against the oracle (shapes, guard bands, in place, the fused forms against the
existing ReLU / add kernels), TEST nets against tests/infer_oracle.py, a TEST net sharing a live Trainer's weights, a TEST Data layer
on an LMDB, `caffe.py test` end to end and the ResNet-50 TEST net.  fp32 math throughout."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from caffe_mpi_b200 import capi, data_api, host_api, lmdb_io
from oracle import layers_oracle as lo
import infer_oracle as io_
import netoracle as no

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SOLVER = 'base_lr: 0.05 lr_policy: "fixed" momentum: 0.9 weight_decay: 0.0005 max_iter: 100 solver_mode: GPU'
ACCURACY = 'layer {{ name: "accuracy" type: "Accuracy" bottom: "{}" bottom: "label" top: "accuracy" }}\n'
GUARD = 64


def _bn_infer(x, gamma, beta, eps, rm, rv, res, y, relu):
    L = capi.lib()
    f = C.c_void_p
    L.b2c_bn_forward_inference.argtypes = [C.c_int, C.c_int, C.c_int, f, f, f, C.c_float, f, f, f, f, C.c_int, f]
    N, Cc = x.shape[0], x.shape[1]
    S = x.numel() // (N * Cc)
    p = lambda t: None if t is None else t.data_ptr()
    rc = L.b2c_bn_forward_inference(N, Cc, S, p(x), p(gamma), p(beta), eps, p(rm), p(rv), p(res), p(y), int(relu), None)
    assert rc == 0, L.b2c_last_error()
    torch.cuda.synchronize()


def _guarded(shape):
    """(whole buffer, view) -- the view sits between two sentinel bands and starts NaN-filled."""
    n = int(np.prod(shape))
    buf = torch.full((n + 2 * GUARD,), 7.25, device="cuda")
    buf[GUARD:GUARD + n] = float("nan")
    return buf, buf[GUARD:GUARD + n].view(shape)


@pytest.mark.parametrize("shape", [(4, 7, 1, 1), (2, 5, 7, 7), (1, 3, 13, 13), (2, 3, 56, 56), (3, 5, 1, 3), (1, 64, 14, 14)])
@pytest.mark.parametrize("affine", [True, False])
def test_bn_inference_kernel_matches_the_oracle(rng, shape, affine):
    Cc = shape[1]
    x = rng.standard_normal(shape).astype(np.float32) * 3 + 1
    rm = rng.uniform(-1, 1, Cc).astype(np.float32)
    rv = rng.uniform(0.2, 3, Cc).astype(np.float32)
    g = rng.uniform(0.5, 1.5, Cc).astype(np.float32) if affine else None
    b = rng.uniform(-0.5, 0.5, Cc).astype(np.float32) if affine else None
    eps = 1e-3
    ref = io_.bn_forward_inference(x, g, b, eps, rm, rv)
    T = lambda a: None if a is None else torch.from_numpy(a).cuda()
    X, G, B, RM, RV = T(x), T(g), T(b), T(rm), T(rv)
    buf, Y = _guarded(shape)
    _bn_infer(X, G, B, eps, RM, RV, None, Y, False)
    got = Y.cpu().numpy()
    assert np.isfinite(got).all()                                             # every element written
    h = buf.cpu().numpy()
    assert (h[:GUARD] == 7.25).all() and (h[-GUARD:] == 7.25).all()          # nothing outside
    assert np.max(np.abs(got - ref)) <= 1e-6 * max(np.max(np.abs(ref)), 1.0)
    Xi = X.clone()                                                            # in place: the same bits
    _bn_infer(Xi, G, B, eps, RM, RV, None, Xi, False)
    assert torch.equal(Xi.view(torch.int32), Y.view(torch.int32))
    # fused forms = the inference kernel, then the existing ReLU / add / add+ReLU kernels
    L = capi.lib()
    for fn in ("b2c_relu_forward", "b2c_add", "b2c_add_relu"):
        getattr(L, fn).argtypes = [C.c_size_t, C.c_void_p, C.c_void_p] + ([C.c_float] if fn == "b2c_relu_forward" else [C.c_void_p]) + [C.c_void_p]
    R = torch.from_numpy(rng.standard_normal(shape).astype(np.float32)).cuda()
    n = X.numel()
    want = torch.empty_like(Y)
    assert L.b2c_relu_forward(n, Y.data_ptr(), want.data_ptr(), 0.0, None) == 0
    _, out = _guarded(shape)
    _bn_infer(X, G, B, eps, RM, RV, None, out, True)
    assert torch.equal(out.view(torch.int32), want.view(torch.int32))
    for relu, fn in ((False, "b2c_add"), (True, "b2c_add_relu")):
        assert getattr(L, fn)(n, Y.data_ptr(), R.data_ptr(), want.data_ptr(), None) == 0
        _bn_infer(X, G, B, eps, RM, RV, R, out, relu)
        assert torch.equal(out.view(torch.int32), want.view(torch.int32)), fn


def _tester_from_model(spec, params, stats, tmp_path, fuse=None, classes=10):
    path = str(tmp_path / "w.caffemodel")
    io_.write_caffemodel(host_api.lib(), path, io_.model_layers(spec, params, stats))
    old = os.environ.get("B2C_FUSE")
    if fuse is not None:
        os.environ["B2C_FUSE"] = "1" if fuse else "0"
    try:
        t = host_api.Tester(no.to_prototxt(spec) + ACCURACY.format(spec[-1]["b"][0]), num_classes=classes)
    finally:
        if fuse is not None:
            os.environ.pop("B2C_FUSE", None) if old is None else os.environ.__setitem__("B2C_FUSE", old)
    t.copy_trained_layers_from(path)
    return t


def _rel(a, ref):
    return float(np.max(np.abs(a.reshape(-1) - ref.reshape(-1))) / max(np.max(np.abs(ref)), 1e-20))


def test_mini_resnet_test_net_matches_the_oracle_and_fusion_changes_no_bit(rng, tmp_path):
    spec = no.mini_resnet()
    params, stats = io_.random_model(spec, rng)
    data = rng.standard_normal(spec[0]["shape"]).astype(np.float32)
    label = rng.integers(0, 10, spec[0]["shape"][0]).astype(np.float32)
    v = io_.forward_test_phase(spec, params, stats, data, label)
    names = [L["n"] for L in spec if L["t"] in ("conv", "pool", "sum", "fc")] + ["conv1/bn", "resA.1.conv2/bn"]
    got = {}
    for fuse in (False, True):
        t = _tester_from_model(spec, params, stats, tmp_path, fuse=fuse)
        t.set_blob("data", data)
        t.set_blob("label", label)
        t.forward()
        blobs = {n: t.get_blob(n) for n in names + ["loss", "accuracy"]}
        for n in names + ["loss"]:
            assert _rel(blobs[n], v[n]) <= 1e-4, (fuse, n)
        assert blobs["accuracy"][0] == lo.accuracy(v["fc"], label)
        got[fuse] = blobs
    for n in [L["n"] for L in spec if L["t"] in ("pool", "fc")] + ["resA.1.sum", "resA.2.sum", "loss", "accuracy"]:
        assert np.array_equal(got[False][n], got[True][n]), n       # B2C_FUSE=0 and the default: the same outputs


def test_mini_inception_test_net_dropout_is_the_identity_and_losses_are_weighted(rng, tmp_path):
    spec = no.mini_inception()
    params, stats = io_.random_model(spec, rng)
    data = rng.standard_normal(spec[0]["shape"]).astype(np.float32)
    label = rng.integers(0, 10, spec[0]["shape"][0]).astype(np.float32)
    v = io_.forward_test_phase(spec, params, stats, data, label)
    t = _tester_from_model(spec, params, stats, tmp_path)
    t.set_blob("data", data)
    t.set_blob("label", label)
    per_batch, means, loss = t.test(1)
    for n in ("conv1", "norm1", "inc/3x3", "inc/5x5", "inc/pool_proj", "inc/output", "aux/fc", "pool5", "cls"):
        assert _rel(t.get_blob(n), v[n]) <= 1e-4, n
    outs = t.outputs()
    assert [(n, round(w, 6)) for n, w, _ in outs] == [("accuracy", 0.0), ("aux/loss1", 0.3), ("loss", 1.0)]
    ref_loss = 0.3 * float(v["aux/loss1"]) + float(v["loss"])
    assert abs(loss - ref_loss) <= 1e-4 * ref_loss
    assert abs(means[1] - float(v["aux/loss1"])) <= 1e-4 * float(v["aux/loss1"])


def _trainer(spec, params):
    t = host_api.Trainer(no.to_prototxt(spec) + ACCURACY.format(spec[-1]["b"][0]), SOLVER, num_classes=10)
    for i, p in enumerate(params):
        t.set_param(i, p)
    return t


def _snapshot_model(t, tmp_path, tag):
    return t.snapshot(str(tmp_path / tag)).replace(".solverstate", ".caffemodel")


def _oracle_scores(spec, model, data, label):
    """(loss, accuracy) of the oracle's TEST forward on the parameters and statistics stored in a .caffemodel"""
    blobs = io_.read_caffemodel(host_api.lib(), model)
    params, stats = [], {}
    for L in spec:
        if L["t"] in ("conv", "fc"):
            params += blobs[L["n"]]
        elif L["t"] == "bn":
            params += blobs[L["n"]][3:5]
            stats[L["n"]] = (blobs[L["n"]][0], blobs[L["n"]][1])
    params = [p.reshape(s) for p, (_, _, s) in zip(params, no.param_shapes(spec))]
    v = io_.forward_test_phase(spec, params, stats, data, label)
    return float(v["loss"]), float(lo.accuracy(v["fc"], label))


def test_test_net_sharing_a_live_trainer(rng, tmp_path):
    """Shared weights: after k steps Test equals the oracle on the trainer's current parameters and running statistics, after k more
    it follows the new weights (a stale conv filter cache fails here), and testing leaves the trainer bit for bit where a trainer
    that never tested would be.  A snapshot loaded with copy-from scores the same bits as the shared net."""
    spec = no.mini_resnet()
    params, _ = io_.random_model(spec, rng)
    data = rng.standard_normal(spec[0]["shape"]).astype(np.float32)
    label = rng.integers(0, 10, spec[0]["shape"][0]).astype(np.float32)
    a, b = _trainer(spec, params), _trainer(spec, params)                  # b never tests
    te = host_api.Tester(no.to_prototxt(spec) + ACCURACY.format("fc"), num_classes=10)
    te.share_trained_layers_with(a)
    te.set_blob("data", data)
    te.set_blob("label", label)
    for t in (a, b):
        t.set_blob("data", data)
        t.set_blob("label", label)
    for rnd in range(2):
        a.step(3)
        b.step(3)
        _, means, loss = te.test(2)
        model = _snapshot_model(a, tmp_path, f"a{rnd}")
        ref_loss, ref_acc = _oracle_scores(spec, model, data, label)
        assert abs(loss - ref_loss) <= 1e-4 * abs(ref_loss), rnd
        assert means[0] == ref_acc
        copied = host_api.Tester(no.to_prototxt(spec) + ACCURACY.format("fc"), num_classes=10)
        copied.copy_trained_layers_from(model)
        copied.set_blob("data", data)
        copied.set_blob("label", label)
        _, m2, l2 = copied.test(2)
        assert l2 == loss and np.array_equal(m2, means)                     # copy-from = shared, bit for bit
    a.step(1)
    b.step(1)
    assert a.loss() == b.loss() and a.iter() == b.iter()
    ma, mb = io_.read_caffemodel(host_api.lib(), _snapshot_model(a, tmp_path, "a")), io_.read_caffemodel(host_api.lib(), _snapshot_model(b, tmp_path, "b"))
    for n in ma:
        for x, y in zip(ma[n], mb[n]):                                      # weights and BatchNorm running statistics
            assert np.array_equal(x, y), n


def test_test_data_layer_reads_the_database_in_order_centre_cropped(rng, tmp_path, monkeypatch):
    monkeypatch.delenv("B2C_DATA", raising=False)
    n, Cc, H, W, crop, B = 7, 3, 9, 11, 5, 3
    imgs = rng.integers(0, 256, (n, Cc, H, W), dtype=np.uint8)
    labels = rng.integers(0, 10, n)
    src = str(tmp_path / "val_lmdb")
    lmdb_io.write_datum_lmdb(src, imgs, labels)
    mean = rng.uniform(90, 130, (1, Cc, H, W)).astype(np.float32)
    mean_path = str(tmp_path / "mean.binaryproto")
    data_api.blobproto_save(mean_path, mean)
    net = ('name: "t"\n'
           'layer { name: "data" type: "Data" top: "data" top: "label" include { phase: TRAIN }\n'
           '  data_param { source: "/nonexistent_train_lmdb" backend: LMDB batch_size: 8 } transform_param { crop_size: 5 mirror: true } }\n'
           f'layer {{ name: "data" type: "Data" top: "data" top: "label" include {{ phase: TEST }}\n'
           f'  data_param {{ source: "{src}" backend: LMDB batch_size: {B} }} transform_param {{ crop_size: {crop} mirror: false mean_file: "{mean_path}" }} }}\n'
           'layer { name: "ip" type: "InnerProduct" bottom: "data" top: "ip" inner_product_param { num_output: 10 weight_filler { type: "gaussian" std: 0.01 } } }\n'
           'layer { name: "loss" type: "SoftmaxWithLoss" bottom: "ip" bottom: "label" top: "loss" }\n')
    t = host_api.Tester(net, num_classes=10)
    h0, w0 = (H - crop) // 2, (W - crop) // 2
    for i in range(5):                                                       # 15 records from a database of 7: wraps twice
        t.forward()
        pos = [(i * B + k) % n for k in range(B)]
        want = lo.transform_u8(imgs[pos], (crop, crop), [h0] * B, [w0] * B, [0] * B, mean_image=mean[0])
        assert np.array_equal(t.get_blob("data").reshape(B, Cc, crop, crop), want), i
        assert np.array_equal(t.get_blob("label"), labels[pos].astype(np.float32)), i
    assert t.database_batches() == 5


def test_caffe_test_end_to_end_equals_the_tester(tmp_path):
    spec = no.mini_resnet()
    net = tmp_path / "net.prototxt"
    net.write_text(no.to_prototxt(spec) + ACCURACY.format("fc"))
    solver = tmp_path / "solver.prototxt"
    solver.write_text(f'net: "{net}"\n' + SOLVER.replace("max_iter: 100", "max_iter: 4") + f'\nsnapshot_prefix: "{tmp_path}/snap"\n')
    run = lambda *a: subprocess.run([sys.executable, os.path.join(ROOT, "tools", "caffe.py"), *a, "--classes=10"], capture_output=True,
                                    text=True, cwd=ROOT)
    r = run("train", f"--solver={solver}")
    assert r.returncode == 0, r.stderr[-2000:]
    model = f"{tmp_path}/snap_iter_4.caffemodel"
    r = run("test", f"--model={net}", f"--weights={model}", "--iterations=3")
    assert r.returncode == 0, r.stderr[-2000:]
    got = [ln.split("caffe.py] ", 1)[1] for ln in r.stdout.splitlines() if "caffe.py] " in ln]
    t = host_api.Tester(str(net), num_classes=10, net_is_text=False)
    t.copy_trained_layers_from(model)
    per_batch, means, loss = t.test(3)
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import caffe as cli
    want = cli.score_lines(t.outputs(), per_batch, means, loss)
    assert got[1:] == want and got[0] == "Running for 3 iterations."


def test_resnet50_test_net_on_the_synthetic_source():
    t = host_api.Tester(os.path.join(HERE, "golden", "reference_models", "models", "resnet50", "train_val.prototxt"), batch=32,
                        net_is_text=False)
    per_batch, means, loss = t.test(2)
    assert np.isfinite(per_batch).all() and np.isfinite(loss)
    names = [n for n, _, _ in t.outputs()]
    for k, n in enumerate(names):
        if n.startswith("accuracy"):
            assert 0.0 <= means[k] <= 1.0

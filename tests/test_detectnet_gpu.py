"""L1Loss kernels per element against tests/detectnet_oracle.py, and the layers DetectNet's TRAIN net adds in whole nets on the
device: L1Loss through TrainNet (both gradient signs, loss_weight 2), and an image database and a float_data label database read by
two Data layers of one net.

Kernels: inputs and outputs in NaN-prefilled buffers with sentinel guard bands (cases.Guarded), aligned and 4 bytes off a 16-byte
boundary; diff = a - b bit for bit; the loss within two float roundings of the float64 sum, and bit-exact where the double sum is
exact; the same bits on a second call; the backward +-alpha or +0 exactly, in place too."""
import numpy as np
import pytest

import detectnet_oracle as dno
from cases import Guarded
from test_data_cpu import oracle_batches

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import caffe_mpi_b200 as m  # noqa: E402
from caffe_mpi_b200 import capi, host_api, lmdb_io  # noqa: E402
from oracle import layers_oracle as lo  # noqa: E402
from test_detectnet_cpu import write_float_lmdb, label_arrays  # noqa: E402

U = 2.0 ** -24
TINY = 1e-44
# one CTA up to 2^19 values, then clusters of 2, 4 and 8 CTAs (loss_cluster_size)
COUNTS = [1, 7, 1000, 78400, (1 << 19) + 5, (1 << 21) + 3, 4 * 10 ** 6 + 1]


def st():
    return capi._stream()


def bits(a):
    return np.ascontiguousarray(a).view(np.int32)


def _inputs(count, seed):
    rng = np.random.default_rng(seed)
    N = 1 if count < 4 else 4
    while count % N:
        N -= 1
    a = (rng.standard_normal(count) * 2).astype(np.float32)
    b = rng.standard_normal(count).astype(np.float32)
    b[::17] = a[::17]                                                   # exact zeros of a - b: sign 0
    return N, a, b


@pytest.mark.parametrize("count", COUNTS)
@pytest.mark.parametrize("off", [0, 1], ids=["aligned", "off4"])
def test_l1_loss_forward_and_backward(count, off):
    N, a, b = _inputs(count, count)
    L = m.lib()
    A, B = Guarded(count, off, a), Guarded(count, off, b)
    out = []
    for _ in range(2):
        D, LS = Guarded(count, off), Guarded(1)
        capi.check(L.b2c_l1_loss_forward(N, count, A.ptr(), B.ptr(), D.ptr(), LS.ptr(), st()))
        out.append((D.read().copy(), LS.read()[0]))
    assert np.array_equal(bits(out[0][0]), bits(out[1][0])) and bits(np.float32(out[0][1])) == bits(np.float32(out[1][1]))
    diff, loss = out[0]
    assert np.array_equal(bits(diff), bits(a - b))
    ref, _ = dno.l1_loss(diff.reshape(N, -1), np.zeros_like(diff).reshape(N, -1))       # |d| summed exactly in float64
    assert abs(float(loss) - ref) <= (2 * U + count * 2.0 ** -53) * ref + TINY, (loss, ref)
    for sign, inplace in ((1.0, False), (-1.0, True)):
        alpha = np.float32(sign * 2.0 / N)
        DD = Guarded(count, off, diff)
        DX = DD if inplace else Guarded(count, off)
        capi.check(L.b2c_l1_loss_backward(count, DD.ptr(), float(alpha), DX.ptr(), st()))
        assert np.array_equal(bits(DX.read()), bits(dno.l1_backward_f32(diff, alpha)))


@pytest.mark.parametrize("count", [5, 4099, (1 << 20) + 1])
def test_l1_loss_is_bit_exact_when_the_sum_is(count):
    """Inputs on a 2^-8 grid below 2^7: every |d| and every partial sum is exact in double, so the loss is fl(fl(S) / N) exactly."""
    rng = np.random.default_rng(count)
    a = (rng.integers(-2 ** 14, 2 ** 14, count) / 256.0).astype(np.float32)
    b = (rng.integers(-2 ** 14, 2 ** 14, count) / 256.0).astype(np.float32)
    N = 5 if count % 5 == 0 else 1
    L = m.lib()
    A, B, D, LS = Guarded(count, 0, a), Guarded(count, 0, b), Guarded(count), Guarded(1)
    capi.check(L.b2c_l1_loss_forward(N, count, A.ptr(), B.ptr(), D.ptr(), LS.ptr(), st()))
    want, _ = dno.l1_loss_f32(a, b, N)
    assert bits(np.float32(LS.read()[0])) == bits(want)


def test_l1_loss_bad_arguments_are_refused():
    L = m.lib()
    X = Guarded(8)
    assert L.b2c_l1_loss_forward(0, 8, X.ptr(), X.ptr(), X.ptr(), X.ptr(), st()) != 0
    assert L.b2c_l1_loss_forward(1, 0, X.ptr(), X.ptr(), X.ptr(), X.ptr(), st()) != 0
    assert L.b2c_l1_loss_forward(1, 8, X.ptr(), None, X.ptr(), X.ptr(), st()) != 0
    assert L.b2c_l1_loss_backward(8, None, 1.0, X.ptr(), st()) != 0


# ------------------------------------------------------------------------------------------------------------ whole nets
def rel(got, ref):
    return float(np.abs(np.asarray(got, np.float64).reshape(-1) - np.asarray(ref).reshape(-1)).max() / max(np.abs(ref).max(), 1e-30))


def test_l1_loss_gradients_through_trainnet_match_oracle():
    """conv(1x1, bias) -> Flatten -> L1Loss (loss_weight 2, DetectNet's) against a target: the conv's gradients are the
    +2 / N * sign(y - t) the loss sends back.  Then the target computed by a second conv, which takes the minus sign."""
    rng = np.random.default_rng(9)
    N, C, O, H, W = 4, 3, 5, 3, 4
    x = rng.standard_normal((N, C, H, W)).astype(np.float32)
    tgt = rng.standard_normal((N, O * H * W)).astype(np.float32)
    w = (rng.standard_normal((O, C, 1, 1)) * 0.5).astype(np.float32)
    b = rng.standard_normal(O).astype(np.float32) * 0.1
    conv = ('layer {{ name: "{n}" type: "Convolution" bottom: "data" top: "{n}" convolution_param {{ num_output: %d kernel_size: 1 '
            'weight_filler {{ type: "msra" }} }} }}\n' % O)
    net = ('name: "l1" layer { name: "data" type: "Input" top: "data" top: "t" input_param { shape { dim: %d dim: %d dim: %d dim: %d } '
           'shape { dim: %d dim: %d } } }\n' % (N, C, H, W, N, O * H * W) + conv.format(n="conv") +
           'layer { name: "flat" type: "Flatten" bottom: "conv" top: "flat" }\n'
           'layer { name: "loss" type: "L1Loss" bottom: "flat" bottom: "t" top: "loss" loss_weight: 2 }\n')
    t = host_api.Trainer(net, 'base_lr: 0.01 lr_policy: "fixed" max_iter: 1', num_classes=10)
    t.set_param(0, w)
    t.set_param(1, b)
    t.set_blob("data", x)
    t.set_blob("t", tgt)
    loss = t.forward_backward()
    y = np.einsum("oc,nchw->nohw", w.reshape(O, C).astype(np.float64), x) + b[None, :, None, None]
    ref_loss, d = dno.l1_loss(y.reshape(N, -1), tgt)
    assert np.abs(d).min() > 1e-4                                       # no element near the kink
    assert abs(loss - ref_loss) <= 1e-5 * ref_loss
    g = dno.l1_backward(d, N, loss_weight=2.0)[0].reshape(N, O, H, W)
    assert rel(t.get_param(0, 1), np.einsum("nohw,nchw->oc", g, x)) <= 1e-5
    assert rel(t.get_param(1, 1), g.sum(axis=(0, 2, 3))) <= 1e-6
    net2 = (net.replace('bottom: "t" top: "loss"', 'bottom: "flat2" top: "loss"').replace(
        'layer { name: "loss"', conv.format(n="conv2") + 'layer { name: "flat2" type: "Flatten" bottom: "conv2" top: "flat2" }\nlayer { name: "loss"'))
    t2 = host_api.Trainer(net2, 'base_lr: 0.01 lr_policy: "fixed" max_iter: 1', num_classes=10)
    w2 = (rng.standard_normal((O, C, 1, 1)) * 0.5).astype(np.float32)
    for i, p in enumerate((w, b, w2, np.zeros(O, np.float32))):
        t2.set_param(i, p)
    t2.set_blob("data", x)
    loss2 = t2.forward_backward()
    y2 = np.einsum("oc,nchw->nohw", w2.reshape(O, C).astype(np.float64), x)
    ref2, d2 = dno.l1_loss(y.reshape(N, -1), y2.reshape(N, -1))
    assert abs(loss2 - ref2) <= 1e-5 * ref2
    g2 = dno.l1_backward(d2, N, loss_weight=2.0)[0].reshape(N, O, H, W)
    assert rel(t2.get_param(0, 1), np.einsum("nohw,nchw->oc", g2, x)) <= 1e-5
    assert rel(t2.get_param(2, 1), -np.einsum("nohw,nchw->oc", g2, x)) <= 1e-5
    assert rel(t2.get_param(3, 1), -g2.sum(axis=(0, 2, 3))) <= 1e-6


IMG_LABEL_NET = ('name: "img_label"\n'
                 'layer {{ name: "data" type: "Data" top: "data" data_param {{ source: "{img}" backend: LMDB batch_size: {B} parser_threads: 2 }} '
                 'transform_param {{ mean_value: 128 scale: 0.0078125 }} }}\n'
                 'layer {{ name: "label" type: "Data" top: "label" data_param {{ source: "{lab}" backend: LMDB batch_size: {B} }} }}\n'
                 'layer {{ name: "ip" type: "InnerProduct" bottom: "data" top: "ip" inner_product_param {{ num_output: {K} '
                 'weight_filler {{ type: "gaussian" std: 0.01 }} }} }}\n'
                 'layer {{ name: "loss" type: "L1Loss" bottom: "ip" bottom: "label" top: "loss" loss_weight: 2 }}\n')


def test_image_and_float_label_databases_feed_one_net(tmp_path, monkeypatch):
    """Two Data layers on the device: uint8 images through the device transform, DIGITS-layout float labels copied verbatim, in step,
    with the L1Loss between an InnerProduct and the labels equal to the float64 oracle on the same batch and weights."""
    monkeypatch.delenv("B2C_DATA", raising=False)
    n, B, steps, max_boxes = 21, 4, 8, 2
    rng = np.random.default_rng(12)
    imgs = rng.integers(0, 256, (n, 3, 6, 5), dtype=np.uint8)
    lmdb_io.write_datum_lmdb(str(tmp_path / "img"), imgs, np.zeros(n, np.int64))
    lab = label_arrays(n, max_boxes, seed=3)
    write_float_lmdb(str(tmp_path / "lab"), lab)
    K = (max_boxes + 1) * 16
    t = host_api.Trainer(IMG_LABEL_NET.format(img=tmp_path / "img", lab=tmp_path / "lab", B=B, K=K),
                         'base_lr: 0.01 lr_policy: "fixed" max_iter: 100', num_classes=10)
    zeros = np.zeros(B, np.int32)
    for i in range(steps):
        w, b = t.get_param(0).copy(), t.get_param(1).copy()
        t.step(1, copy_input=True)
        pos = [p for p, _ in oracle_batches(n, steps, B, 1, 0, 2)[i]]
        x = t.get_blob("data").reshape(B, 3, 6, 5)
        assert np.array_equal(x, lo.transform_u8(imgs[pos], (6, 5), zeros, zeros, zeros, [128.0] * 3, None, 0.0078125)), f"data of batch {i}"
        assert np.array_equal(bits(t.get_blob("label").reshape(B, 1, max_boxes + 1, 16)), bits(lab[pos])), f"labels of batch {i}"
        y = x.reshape(B, -1).astype(np.float64) @ w.reshape(K, -1).T.astype(np.float64) + b
        ref, _ = dno.l1_loss(y, lab[pos].reshape(B, -1))
        assert abs(t.loss() - ref) <= 1e-5 * ref, (i, t.loss(), ref)
    assert t.database_batches() == steps

"""Softmax, Sigmoid, SigmoidCrossEntropyLoss and EuclideanLoss kernels per element against the float64 forms of
tests/newlayers_oracle.py, and the layers in whole nets through TrainNet.

Per kernel: inputs and outputs in NaN-prefilled buffers with sentinel guard bands (cases.Guarded); every element within a stated
c * 2^-24 * sum|terms| bound; the same bits on a second call; in place where the entry point allows it; 4 bytes off a 16-byte
boundary (the scalar path).  Then the bit-for-bit relations b2c.h promises, the autoencoder-shaped net against the net oracle
(loss, every parameter gradient, three steps of Nesterov / AdaGrad / AdaDelta), and a deploy form scored on trained weights."""
import numpy as np
import pytest

import newlayers_oracle as nlo
from cases import Guarded

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import caffe_mpi_b200 as m  # noqa: E402
from caffe_mpi_b200 import capi, host_api  # noqa: E402
import solver_oracle as so  # noqa: E402

U = 2.0 ** -24
TINY = 1e-44


def st():
    return capi._stream()


def bits(a):
    return np.ascontiguousarray(a).view(np.int32)


def within(got, ref, bound, what):
    err = np.abs(got.astype(np.float64) - ref)
    bad = np.flatnonzero(~(err <= bound))
    assert bad.size == 0, f"{what}: {bad.size} elements out of bound, first {bad[:5]}: got {got.reshape(-1)[bad[:3]]} ref {ref.reshape(-1)[bad[:3]]}"


# ------------------------------------------------------------------------------------------------------------ Softmax
SOFTMAX = [(4, 1, 1), (4, 10, 1), (3, 1000, 1), (2, 21841, 1), (257, 10, 1), (2, 21, 49), (2, 21, 7 * 8), (3, 5, 3), (1, 1, 6)]


@pytest.mark.parametrize("outer,C,inner", SOFTMAX, ids=[f"{o}x{c}x{i}" for o, c, i in SOFTMAX])
@pytest.mark.parametrize("off", [0, 1], ids=["aligned", "off4"])
@pytest.mark.parametrize("inplace", [False, True], ids=["out", "inplace"])
def test_softmax_per_element(outer, C, inner, off, inplace):
    rng = np.random.default_rng(outer * 7 + C + inner)
    shape = (outer, C, inner)
    x = (rng.standard_normal(shape) * 3).astype(np.float32)
    dy = rng.standard_normal(shape).astype(np.float32)
    L = m.lib()
    runs = []
    for _ in range(2):
        X = Guarded(x.size, off, x)
        Y = X if inplace else Guarded(x.size, off)
        capi.check(L.b2c_softmax_forward(outer, C, inner, X.ptr(), Y.ptr(), st()))
        y = Y.read().reshape(shape).copy()
        YY = Guarded(y.size, off, y)
        DY = Guarded(dy.size, off, dy)
        DX = DY if inplace else Guarded(dy.size, off)
        capi.check(L.b2c_softmax_backward(outer, C, inner, YY.ptr(), DY.ptr(), DX.ptr(), st()))
        runs.append((y, DX.read().reshape(shape).copy()))
    (y, dx), (y2, dx2) = runs
    assert np.array_equal(bits(y), bits(y2)) and np.array_equal(bits(dx), bits(dx2))
    x64 = x.astype(np.float64)
    ref = nlo.softmax_forward(x64, 1)
    shift = np.abs(x64 - x64.max(axis=1, keepdims=True))
    # expf (2 ulp), the channel sum (C - 1 roundings), the division and the scale; the rounding of x - max scales with |x - max|
    within(y, ref, (C + 8 + shift) * U * ref + TINY, "y")
    y64, d64 = y.astype(np.float64), dy.astype(np.float64)
    ref_dx = nlo.softmax_backward(y64, d64, 1)
    dot = (d64 * y64).sum(axis=1, keepdims=True)
    S = np.abs(d64 * y64).sum(axis=1, keepdims=True)
    within(dx, ref_dx, (C + 4) * U * (S + np.abs(d64) + np.abs(dot)) * y64 + TINY, "dx")


@pytest.mark.parametrize("N,C", [(4, 10), (3, 1000), (2, 21841), (257, 10)])
def test_softmax_rows_equal_softmax_loss_prob(N, C):
    """inner == 1: the Softmax top is SoftmaxWithLoss's prob, bit for bit."""
    rng = np.random.default_rng(C)
    x = (rng.standard_normal((N, C)) * 3).astype(np.float32)
    lab = rng.integers(0, C, N).astype(np.float32)
    X, Y, P, LB, LS = Guarded(x.size, 0, x), Guarded(x.size), Guarded(x.size), Guarded(N, 0, lab), Guarded(1)
    capi.check(m.lib().b2c_softmax_forward(N, C, 1, X.ptr(), Y.ptr(), st()))
    capi.check(m.lib().b2c_softmax_loss_forward(N, C, X.ptr(), LB.ptr(), P.ptr(), LS.ptr(), st()))
    assert np.array_equal(bits(Y.read()), bits(P.read()))


# ------------------------------------------------------------------------------------------------------------ Sigmoid
SIZES = [1, 3, 1000, 78400, 524291]


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("off", [0, 1], ids=["aligned", "off4"])
@pytest.mark.parametrize("inplace", [False, True], ids=["out", "inplace"])
def test_sigmoid_per_element(n, off, inplace):
    rng = np.random.default_rng(n)
    x = (rng.standard_normal(n) * 4).astype(np.float32)
    dy = rng.standard_normal(n).astype(np.float32)
    L = m.lib()
    runs = []
    for _ in range(2):
        X = Guarded(n, off, x)
        Y = X if inplace else Guarded(n, off)
        capi.check(L.b2c_sigmoid_forward(n, X.ptr(), Y.ptr(), st()))
        y = Y.read().copy()
        YY, DY = Guarded(n, off, y), Guarded(n, off, dy)
        DX = DY if inplace else Guarded(n, off)
        capi.check(L.b2c_sigmoid_backward(n, YY.ptr(), DY.ptr(), DX.ptr(), st()))
        runs.append((y, DX.read().copy()))
    (y, dx), (y2, dx2) = runs
    assert np.array_equal(bits(y), bits(y2)) and np.array_equal(bits(dx), bits(dx2))
    ref = nlo.sigmoid_forward(x)
    within(y, ref, 6 * U * ref + TINY, "y")                         # expf, the add, the division
    ref_dx = nlo.sigmoid_backward(y.astype(np.float64), dy)
    within(dx, ref_dx, 4 * U * np.abs(ref_dx) + TINY, "dx")


# ------------------------------------------------------------------------------------------------------------ losses
LOSS_COUNTS = [1, 3, 1000, 78400, 2 * (1 << 18) + 3, 10 ** 7]      # around the cluster-size steps (one CTA per 256K values)


def _loss_inputs(count, seed):
    rng = np.random.default_rng(seed)
    N = 100 if count % 100 == 0 else 1                            # (the loss divides by the first axis)
    x = (rng.standard_normal(count) * 4).astype(np.float32)
    t = rng.uniform(0, 1, count).astype(np.float32)
    return N, x, t


@pytest.mark.parametrize("count", LOSS_COUNTS)
@pytest.mark.parametrize("off", [0, 1], ids=["aligned", "off4"])
def test_sigmoid_ce_loss(count, off):
    N, x, t = _loss_inputs(count, count)
    L = m.lib()
    X, T = Guarded(count, off, x), Guarded(count, off, t)
    out = []
    for _ in range(2):
        LS = Guarded(1)
        capi.check(L.b2c_sigmoid_ce_loss_forward(N, count, X.ptr(), T.ptr(), LS.ptr(), st()))
        out.append(LS.read()[0])
    assert bits(np.float32(out[0])) == bits(np.float32(out[1]))
    ref = nlo.sigmoid_ce_loss(x.reshape(N, -1), t.reshape(N, -1))
    x64, t64 = x.astype(np.float64), t.astype(np.float64)
    pos = (x64 >= 0)
    terms = np.abs(x64 * (t64 - pos)) + np.abs(np.log1p(np.exp(x64 - 2 * x64 * pos))) + 1.0
    assert abs(out[0] - ref) <= 6 * U * terms.sum() / N + 3 * U * abs(ref), (out[0], ref)
    # backward, in place and out of place
    lw = 0.7
    scale = np.float32(lw / N)
    for inplace in (False, True):
        XX = Guarded(count, off, x)
        DX = XX if inplace else Guarded(count, off)
        capi.check(L.b2c_sigmoid_ce_loss_backward(count, XX.ptr(), T.ptr(), float(scale), DX.ptr(), st()))
        dx = DX.read()
        sig = nlo.sigmoid_forward(x64)
        ref_dx = (sig - t64) * np.float64(scale)
        within(dx, ref_dx, (6 * U * sig + 2 * U * np.abs(sig - t64)) * float(scale) + TINY, "dx")


@pytest.mark.parametrize("count", [1, 1000, 78400, 10 ** 6 + 1])
def test_sigmoid_ce_backward_is_sigmoid_forward_minus_target_times_scale(count):
    """b2c.h: the backward's sigmoid is b2c_sigmoid_forward's expression.  (sigmoid_forward(x) - t) * scale, formed with the public
    Euclidean kernels (diff = a - b, then alpha * diff), gives the same bits."""
    _, x, t = _loss_inputs(count, count + 1)
    L = m.lib()
    scale = float(np.float32(1.0 / 100))
    X, T = Guarded(count, 0, x), Guarded(count, 0, t)
    S, D, LS, R, G = Guarded(count), Guarded(count), Guarded(1), Guarded(count), Guarded(count)
    capi.check(L.b2c_sigmoid_forward(count, X.ptr(), S.ptr(), st()))
    capi.check(L.b2c_euclidean_loss_forward(1, count, S.ptr(), T.ptr(), D.ptr(), LS.ptr(), st()))
    capi.check(L.b2c_euclidean_loss_backward(count, D.ptr(), scale, R.ptr(), st()))
    capi.check(L.b2c_sigmoid_ce_loss_backward(count, X.ptr(), T.ptr(), scale, G.ptr(), st()))
    assert np.array_equal(bits(G.read()), bits(R.read()))


@pytest.mark.parametrize("count", LOSS_COUNTS)
@pytest.mark.parametrize("off", [0, 1], ids=["aligned", "off4"])
def test_euclidean_loss(count, off):
    N, a, _ = _loss_inputs(count, count + 2)
    b = np.random.default_rng(count + 3).standard_normal(count).astype(np.float32)
    L = m.lib()
    A, B = Guarded(count, off, a), Guarded(count, off, b)
    out = []
    for _ in range(2):
        D, LS = Guarded(count, off), Guarded(1)
        capi.check(L.b2c_euclidean_loss_forward(N, count, A.ptr(), B.ptr(), D.ptr(), LS.ptr(), st()))
        out.append((D.read().copy(), LS.read()[0]))
    assert np.array_equal(bits(out[0][0]), bits(out[1][0])) and bits(np.float32(out[0][1])) == bits(np.float32(out[1][1]))
    diff, loss = out[0]
    ref, d64 = nlo.euclidean_loss(a.reshape(N, -1), b.reshape(N, -1))
    within(diff, d64.reshape(-1), U * np.abs(d64.reshape(-1)) + TINY, "diff")
    assert abs(loss - ref) <= 6 * U * ref + TINY, (loss, ref)
    for sign, inplace in ((1.0, False), (-1.0, True)):
        alpha = np.float32(sign * 0.5 / N)
        DD = Guarded(count, off, diff)
        DX = DD if inplace else Guarded(count, off)
        capi.check(L.b2c_euclidean_loss_backward(count, DD.ptr(), float(alpha), DX.ptr(), st()))
        ref_dx = diff.astype(np.float64) * np.float64(alpha)
        within(DX.read(), ref_dx, U * np.abs(ref_dx) + TINY, "dx")


def test_bad_arguments_are_refused():
    L = m.lib()
    X = Guarded(8)
    assert L.b2c_softmax_forward(0, 4, 1, X.ptr(), X.ptr(), st()) != 0
    assert L.b2c_softmax_backward(1, 4, 0, X.ptr(), X.ptr(), X.ptr(), st()) != 0
    assert L.b2c_sigmoid_ce_loss_forward(0, 8, X.ptr(), X.ptr(), X.ptr(), st()) != 0
    assert L.b2c_euclidean_loss_forward(1, 0, X.ptr(), X.ptr(), X.ptr(), X.ptr(), st()) != 0
    assert L.b2c_sigmoid_forward(8, None, X.ptr(), st()) != 0


# ------------------------------------------------------------------------------------------------------------ whole nets
def _trainer(spec, solver, rng):
    t = host_api.Trainer(nlo.to_prototxt(spec), solver, num_classes=10)
    params = []
    for i, (_, kind, shp) in enumerate(nlo.param_shapes(spec)):
        p = (rng.standard_normal(shp) * np.sqrt(1.0 / shp[1])).astype(np.float32) if kind == "w" else \
            rng.uniform(-0.2, 0.2, shp).astype(np.float32)
        t.set_param(i, p)
        params.append(p)
    data = rng.uniform(0, 1, spec[0]["shape"]).astype(np.float32)
    t.set_blob("data", data)
    return t, params, data


def rel(a, ref, floor=1e-20):
    return float(np.max(np.abs(a.reshape(-1) - ref.reshape(-1))) / max(np.max(np.abs(ref)), floor))


def test_autoencoder_loss_and_gradients_match_oracle():
    spec = nlo.autoencoder()
    t, params, data = _trainer(spec, 'base_lr: 0.01 lr_policy: "fixed" max_iter: 10', np.random.default_rng(1701))
    loss = t.forward_backward()
    ref_loss, grads, v = nlo.forward_backward(spec, params, data)
    assert abs(loss - ref_loss) <= 1e-4 * abs(ref_loss), (loss, ref_loss)
    for i, g in enumerate(grads):
        assert rel(t.get_param(i, 1), g) <= 1e-4, i
    # the weight-0 branch ran forward: its loss blob holds the Euclidean loss of sigmoid(decode1) against the flattened input
    assert abs(float(t.get_blob("l2_error")[0]) - v["l2_error"]) <= 1e-4 * v["l2_error"]
    assert rel(t.get_blob("flatdata"), data.reshape(data.shape[0], -1)) == 0.0
    names = [l[0] for l in t.layers()]
    assert names.count("loss") == 2


AE_SOLVERS = {     # the reference autoencoder solvers' hyperparameters (examples/mnist/mnist_autoencoder_solver_*.prototxt)
    "Nesterov": (0.01, dict(momentum=0.95, delta=1e-8, rms_decay=0.0, momentum2=0.999)),
    "AdaGrad": (0.01, dict(momentum=0.0, delta=1e-8, rms_decay=0.0, momentum2=0.999)),
    "AdaDelta": (1.0, dict(momentum=0.95, delta=1e-8, rms_decay=0.0, momentum2=0.999)),
}


@pytest.mark.parametrize("kind", list(AE_SOLVERS))
def test_autoencoder_steps_match_oracle(kind):
    base_lr, hp = AE_SOLVERS[kind]
    solver = ('type: "%s" base_lr: %g lr_policy: "fixed" momentum: %g delta: %g weight_decay: 0.0005 max_iter: 100'
              % (kind, base_lr, hp["momentum"], hp["delta"]))
    spec = nlo.autoencoder()
    t, params, data = _trainer(spec, solver, np.random.default_rng(7))
    shapes = nlo.param_shapes(spec)
    ref = [p.copy() for p in params]
    hist = [np.zeros(p.size, np.float32) for p in params]
    hist2 = [np.zeros(p.size, np.float32) for p in params]
    losses, ref_losses = [], []
    for it in range(3):
        loss, grads, _ = nlo.forward_backward(spec, ref, data)
        ref_losses.append(loss)
        for i, g in enumerate(grads):
            decay = 0.0005 * (1.0 if shapes[i][1] == "w" else 0.0)
            _, w, hist[i], h2 = so.update(kind, g.astype(np.float32), ref[i], hist[i], hist2[i], hp, base_lr, decay, t=it + 1)
            ref[i] = np.asarray(w, np.float32).reshape(ref[i].shape)
            if h2 is not None:
                hist2[i] = h2
        t.step(1)
        losses.append(t.loss())
    np.testing.assert_allclose(losses, ref_losses, rtol=1e-4)
    for i in range(len(ref)):
        assert rel(t.get_param(i, 0), ref[i]) <= 1e-4, (kind, i)


def _convnet(head, batch=4):
    """conv -> relu -> conv(classes) -> global AVE pool -> logits [N, C]; TRAIN ends in SoftmaxWithLoss, the deploy form in Softmax,
    and the `chan` head adds a Softmax over the channels of the second conv (inner = H * W > 1)."""
    s = 'name: "mini_deploy"\n'
    if head == "train":
        s += ('layer { name: "data" type: "Input" top: "data" top: "label" input_param { shape { dim: %d dim: 3 dim: 8 dim: 8 } '
              'shape { dim: %d } } }\n' % (batch, batch))
    else:
        s += 'layer { name: "data" type: "Input" top: "data" input_param { shape { dim: %d dim: 3 dim: 8 dim: 8 } } }\n' % batch
    s += ('layer { name: "conv1" type: "Convolution" bottom: "data" top: "conv1" convolution_param { num_output: 8 kernel_size: 3 pad: 1 '
          'weight_filler { type: "msra" } } }\n'
          'layer { name: "relu1" type: "ReLU" bottom: "conv1" top: "conv1" }\n'
          'layer { name: "conv2" type: "Convolution" bottom: "conv1" top: "conv2" convolution_param { num_output: 5 kernel_size: 1 '
          'weight_filler { type: "msra" } } }\n'
          'layer { name: "pool" type: "Pooling" bottom: "conv2" top: "logits" pooling_param { pool: AVE global_pooling: true } }\n'
          'layer { name: "flat" type: "Flatten" bottom: "logits" top: "flat" }\n')
    if head == "train":
        s += 'layer { name: "loss" type: "SoftmaxWithLoss" bottom: "flat" bottom: "label" top: "loss" }\n'
    else:
        s += 'layer { name: "prob" type: "Softmax" bottom: "flat" top: "prob" }\n'
        s += 'layer { name: "chanprob" type: "Softmax" bottom: "conv2" top: "chanprob" softmax_param { axis: -3 } }\n'
    return s


def test_deploy_form_scores_trained_weights(tmp_path):
    """A net trained and snapshotted here, then its deploy form (Input -> ... -> Softmax) loaded with the weights: prob equals the
    softmax of the TRAIN net's logits on the same input, and the channel softmax (inner = 64) matches the oracle."""
    rng = np.random.default_rng(11)
    t = host_api.Trainer(_convnet("train"), 'base_lr: 0.05 lr_policy: "fixed" momentum: 0.9 max_iter: 100', num_classes=5)
    data = rng.standard_normal((4, 3, 8, 8)).astype(np.float32)
    t.set_blob("data", data)
    t.set_blob("label", rng.integers(0, 5, 4).astype(np.float32))
    t.step(5)
    state = t.snapshot(str(tmp_path / "mini"))
    t.forward_backward()
    logits = t.get_blob("flat").reshape(4, 5).astype(np.float64)
    te = host_api.Tester(_convnet("deploy"), num_classes=5)
    assert te.copy_trained_layers_from(state.replace(".solverstate", ".caffemodel")) == 2
    te.set_blob("data", data)
    te.forward()
    prob = te.get_blob("prob").reshape(4, 5)
    assert rel(prob, nlo.softmax_forward(logits, 1)) <= 1e-5
    conv2 = te.get_blob("conv2").reshape(4, 5, 8, 8)
    assert rel(te.get_blob("chanprob").reshape(4, 5, 8, 8), nlo.softmax_forward(conv2.astype(np.float64), 1)) <= 1e-5


def test_sigmoid_ce_refuses_a_target_that_needs_a_gradient():
    """sigmoid_cross_entropy_loss_layer.cpp:52-55: the target bottom cannot take a gradient -- here refused when the net is built."""
    net = ('name: "bad" layer { name: "data" type: "Input" top: "data" input_param { shape { dim: 4 dim: 6 } } }\n'
           'layer { name: "a" type: "InnerProduct" bottom: "data" top: "a" inner_product_param { num_output: 3 } }\n'
           'layer { name: "b" type: "InnerProduct" bottom: "data" top: "b" inner_product_param { num_output: 3 } }\n'
           'layer { name: "loss" type: "SigmoidCrossEntropyLoss" bottom: "a" bottom: "b" top: "loss" }\n')
    with pytest.raises(host_api.HostError, match="SigmoidCrossEntropyLoss Layer cannot backpropagate to label inputs."):
        host_api.Trainer(net, 'base_lr: 0.01 lr_policy: "fixed" max_iter: 1', num_classes=10)
    # the same net with a data-fed target builds
    ok = net.replace('bottom: "b" top: "loss"', 'bottom: "t" top: "loss"').replace(
        'top: "data" input_param { shape { dim: 4 dim: 6 } }', 'top: "data" top: "t" input_param { shape { dim: 4 dim: 6 } shape { dim: 4 dim: 3 } }')
    host_api.Trainer(ok, 'base_lr: 0.01 lr_policy: "fixed" max_iter: 1', num_classes=10)


def test_flatten_backward_and_euclidean_gradients_match_oracle():
    """conv(1x1, bias) -> Flatten -> EuclideanLoss (loss_weight 2) against a target: the conv's weight and bias gradients reach it only
    through Flatten's backward copy and EuclideanLoss's +alpha * diff.  Then the same with the target computed by a second conv, which
    takes -alpha * diff."""
    rng = np.random.default_rng(5)
    N, C, O, H, W = 4, 3, 5, 3, 4
    x = rng.standard_normal((N, C, H, W)).astype(np.float32)
    tgt = rng.standard_normal((N, O * H * W)).astype(np.float32)
    w = (rng.standard_normal((O, C, 1, 1)) * 0.5).astype(np.float32)
    b = rng.standard_normal(O).astype(np.float32) * 0.1
    conv = ('layer {{ name: "{n}" type: "Convolution" bottom: "data" top: "{n}" convolution_param {{ num_output: %d kernel_size: 1 '
            'weight_filler {{ type: "msra" }} }} }}\n' % O)
    net = ('name: "flat" layer { name: "data" type: "Input" top: "data" top: "t" input_param { shape { dim: %d dim: %d dim: %d dim: %d } '
           'shape { dim: %d dim: %d } } }\n' % (N, C, H, W, N, O * H * W) + conv.format(n="conv") +
           'layer { name: "flat" type: "Flatten" bottom: "conv" top: "flat" }\n'
           'layer { name: "loss" type: "EuclideanLoss" bottom: "flat" bottom: "t" top: "loss" loss_weight: 2 }\n')
    t = host_api.Trainer(net, 'base_lr: 0.01 lr_policy: "fixed" max_iter: 1', num_classes=10)
    t.set_param(0, w)
    t.set_param(1, b)
    t.set_blob("data", x)
    t.set_blob("t", tgt)
    loss = t.forward_backward()
    y = np.einsum("oc,nchw->nohw", w.reshape(O, C).astype(np.float64), x) + b[None, :, None, None]
    d = y.reshape(N, -1) - tgt
    ref_loss, _ = nlo.euclidean_loss(y.reshape(N, -1), tgt)
    assert abs(loss - ref_loss) <= 1e-5 * ref_loss                     # the top is the unweighted loss; the weight scales the gradient
    g = (2.0 / N * d).reshape(N, O, H, W)
    assert rel(t.get_param(0, 1), np.einsum("nohw,nchw->oc", g, x)) <= 1e-4
    assert rel(t.get_param(1, 1), g.sum(axis=(0, 2, 3))) <= 1e-4
    assert rel(t.get_blob("flat"), y.reshape(N, -1)) <= 1e-5
    # target from a second conv: its gradient carries the minus sign
    net2 = (net.replace('bottom: "t" top: "loss"', 'bottom: "flat2" top: "loss"') .replace(
        'layer { name: "loss"', conv.format(n="conv2") + 'layer { name: "flat2" type: "Flatten" bottom: "conv2" top: "flat2" }\nlayer { name: "loss"'))
    t2 = host_api.Trainer(net2, 'base_lr: 0.01 lr_policy: "fixed" max_iter: 1', num_classes=10)
    w2 = (rng.standard_normal((O, C, 1, 1)) * 0.5).astype(np.float32)
    for i, p in enumerate((w, b, w2, np.zeros(O, np.float32))):
        t2.set_param(i, p)
    t2.set_blob("data", x)
    t2.forward_backward()
    y2 = np.einsum("oc,nchw->nohw", w2.reshape(O, C).astype(np.float64), x)
    g2 = (2.0 / N * (y - y2)).reshape(N, O, H, W)
    assert rel(t2.get_param(0, 1), np.einsum("nohw,nchw->oc", g2, x)) <= 1e-4
    assert rel(t2.get_param(2, 1), -np.einsum("nohw,nchw->oc", g2, x)) <= 1e-4
    assert rel(t2.get_param(3, 1), -g2.sum(axis=(0, 2, 3))) <= 1e-4

"""Softmax, Sigmoid, Flatten, SigmoidCrossEntropyLoss and EuclideanLoss on the CPU: the float64 forms pinned to the closed forms
and known answers of the reference's own layer tests and to finite differences; the reference's model files that use them
parsed by the host layer (shapes, need-backward with loss pruning, the reported loss blob); the reference's shape errors."""
import os

import numpy as np
import pytest

import newlayers_oracle as nlo

REF = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_models")


def _fd(f, x, eps=1e-6):
    g = np.zeros_like(x)
    for i in np.ndindex(x.shape):
        xp, xm = x.copy(), x.copy()
        xp[i] += eps
        xm[i] -= eps
        g[i] = (f(xp) - f(xm)) / (2 * eps)
    return g


# ---------------------------------------------------------------------------------------------------- oracle pins
def test_softmax_columns_sum_to_one_and_equal_exp_over_sum():
    """test_softmax_layer.cpp TestForward: every (n, spatial) column sums to 1 and equals exp(x) / sum exp(x)."""
    x = np.random.default_rng(0).standard_normal((2, 10, 2, 3))
    y = nlo.softmax_forward(x, axis=1)
    assert np.allclose(y.sum(axis=1), 1.0, atol=1e-12)
    assert np.allclose(y, np.exp(x) / np.exp(x).sum(axis=1, keepdims=True), rtol=1e-12)
    y_neg = nlo.softmax_forward(x, axis=-3)
    assert np.array_equal(y, y_neg)


@pytest.mark.parametrize("shape,axis", [((3, 5), 1), ((2, 4, 3, 2), 1), ((2, 3, 4), -1)])
def test_softmax_backward_matches_finite_differences(shape, axis):
    rng = np.random.default_rng(1)
    x, w = rng.standard_normal(shape), rng.standard_normal(shape)
    y = nlo.softmax_forward(x, axis)
    g = nlo.softmax_backward(y, w, axis)
    assert np.allclose(g, _fd(lambda z: (nlo.softmax_forward(z, axis) * w).sum(), x), atol=1e-7)


def test_sigmoid_closed_form_and_gradient():
    """test_neuron_layer.cpp TestSigmoid: y = 1 / (1 + exp(-x)), in (0, 1); the gradient by finite differences."""
    x = np.random.default_rng(2).standard_normal((2, 3, 4, 5)) * 3
    y = nlo.sigmoid_forward(x)
    assert np.allclose(y, 1.0 / (1.0 + np.exp(-x))) and np.all((y > 0) & (y < 1))
    w = np.random.default_rng(3).standard_normal(x.shape)
    assert np.allclose(nlo.sigmoid_backward(y, w), _fd(lambda z: (nlo.sigmoid_forward(z) * w).sum(), x), atol=1e-7)


def _reference_sigmoid_ce(x, t):
    """test_sigmoid_cross_entropy_loss_layer.cpp's own reference: -sum [t log p + (1 - t) log(1 - p)] / num, p = sigmoid(x)."""
    p = 1.0 / (1.0 + np.exp(-x))
    return -np.sum(t * np.log(p) + (1 - t) * np.log(1 - p)) / x.shape[0]


def test_sigmoid_ce_loss_equals_the_reference_tests_loss():
    rng = np.random.default_rng(4)
    for scale in (1.0, 4.0, 10.0):
        x = rng.standard_normal((10, 5, 1, 1)) * scale
        t = rng.uniform(0, 1, x.shape)
        assert nlo.sigmoid_ce_loss(x, t) == pytest.approx(_reference_sigmoid_ce(x, t), rel=1e-7)   # (the naive form loses digits in log(1 - p))
    # the stable form does not overflow where the naive one does
    assert np.isfinite(nlo.sigmoid_ce_loss(np.array([[800.0, -800.0]]), np.array([[0.0, 1.0]])))
    assert nlo.sigmoid_ce_loss(np.array([[800.0, -800.0]]), np.array([[0.0, 1.0]])) == pytest.approx(1600.0)


def test_sigmoid_ce_gradient_matches_finite_differences():
    rng = np.random.default_rng(5)
    x, t = rng.standard_normal((4, 6)), rng.uniform(0, 1, (4, 6))
    g = nlo.sigmoid_ce_backward(x, t, loss_weight=0.7)
    assert np.allclose(g, _fd(lambda z: 0.7 * nlo.sigmoid_ce_loss(z, t), x), atol=1e-7)


def test_euclidean_loss_known_answer_and_gradients():
    """test_euclidean_loss_layer.cpp: loss = sum (a - b)^2 / num / 2; gradients +-diff / num, by finite differences."""
    rng = np.random.default_rng(6)
    a, b = rng.standard_normal((10, 5, 1, 1)), rng.standard_normal((10, 5, 1, 1))
    loss, d = nlo.euclidean_loss(a, b)
    assert loss == pytest.approx(np.sum((a - b) ** 2) / 10 / 2, rel=1e-12)
    ga, gb = nlo.euclidean_backward(d, 10, loss_weight=2.0)
    assert np.allclose(ga, _fd(lambda z: 2.0 * nlo.euclidean_loss(z, b)[0], a), atol=1e-7)
    assert np.allclose(gb, _fd(lambda z: 2.0 * nlo.euclidean_loss(a, z)[0], b), atol=1e-7)


@pytest.mark.parametrize("shape,axis,end,want", [
    ((2, 3, 6, 5), 1, -1, (2, 90)),            # test_flatten_layer.cpp TestSetup
    ((2, 3, 6, 5), 2, -1, (2, 3, 30)),         # TestSetupWithAxis
    ((2, 3, 6, 5), 0, 1, (6, 6, 5)),           # TestSetupWithEndAxis
    ((2, 3, 6, 5), 0, -1, (180,)),             # TestSetupWithStartAndEndAxis
])
def test_flatten_shapes(shape, axis, end, want):
    assert nlo.flatten_shape(shape, axis, end) == want


# ---------------------------------------------------------------------------------------------------- the host layer's graph
def _net(text_or_path, phase="TRAIN", is_text=False, **kw):
    from caffe_mpi_b200 import host_api as h
    return h.Net(text_or_path, phase, is_text=is_text, **kw)


def test_autoencoder_train_net_parses_with_pruning_and_loss_blob():
    n = _net(os.path.join(REF, "examples/mnist/mnist_autoencoder.prototxt"), default_channels=1, default_size=28)
    layers = n.layers()
    names = [l[0] for l in layers]
    assert names == ["data", "flatdata", "encode1", "encode1neuron", "encode2", "encode2neuron", "encode3", "encode3neuron", "encode4",
                     "decode4", "decode4neuron", "decode3", "decode3neuron", "decode2", "decode2neuron", "decode1", "loss",
                     "decode1neuron", "loss"]
    assert [l[1] for l in layers][-3:] == ["SigmoidCrossEntropyLoss", "Sigmoid", "EuclideanLoss"]
    shapes = {l[0]: l[2] for l in layers}
    assert shapes["flatdata"] == (100, 784) and shapes["encode4"] == (100, 30) and shapes["decode1"] == (100, 784)
    plan = dict(zip(range(len(names)), n.backward_plan()))
    by = {names[i]: plan[i] for i in plan if names[i] != "loss"}
    assert by["decode1neuron"] == (False, [False])                     # only feeds the loss_weight 0 EuclideanLoss
    assert plan[len(names) - 1] == (False, [False, False])             # the EuclideanLoss itself
    assert plan[len(names) - 3] == (True, [True, False])               # SigmoidCrossEntropyLoss: gradient to the logits only
    assert by["flatdata"] == (False, [False]) and by["data"] == (False, [])
    assert by["encode1"] == (True, [False]) and by["decode1"] == (True, [True])
    assert n.loss_blob() == "cross_entropy_loss"


def test_existing_nets_keep_their_loss_blob_and_backward_plan():
    """Pruning changes no layer of the training nets that ran before these layer types existed; GoogLeNet reports its main classifier's loss (weight 1)."""
    n = _net(os.path.join(REF, "models/bvlc_googlenet/train_val.prototxt"), batch_override=2)
    assert n.loss_blob() == "loss"
    for (name, ty, _), (nb, pd) in zip(n.layers(), n.backward_plan()):
        if ty in ("Data", "Input"):
            assert not nb
        elif ty == "Accuracy":
            assert not nb
        else:
            assert nb, name
    from caffe_mpi_b200 import models
    for name in ("resnet50", "alexnet", "vgg16", "lenet"):
        g = _net(models.PROTOTXT[name](4), is_text=True, **(dict(default_channels=1, default_size=28) if name == "lenet" else {}))
        for (lname, ty, _), (nb, pd) in zip(g.layers(), g.backward_plan()):
            assert nb == (ty not in ("Data", "Input", "Accuracy")), (name, lname)
        assert g.loss_blob() == [l[0] for l in g.layers() if l[1] == "SoftmaxWithLoss"][-1] or g.loss_blob() == "loss"


def _bottoms(path):
    """layer name -> its first bottom, from the text (the classifier a Softmax reads)."""
    import re
    out = {}
    for block in re.split(r"\blayer\s*\{", open(path).read())[1:]:
        nm, bt = re.search(r'name:\s*"([^"]+)"', block), re.search(r'bottom:\s*"([^"]+)"', block)
        if nm and bt:
            out[nm.group(1)] = bt.group(1)
    return out


def test_inception_v2_test_net_builds_with_softmax_probs():
    n = _net(os.path.join(REF, "models/inception_v2/train_val.prototxt"), "TEST", batch_override=4)
    layers = n.layers()
    shapes = {l[0]: l[2] for l in layers}
    probs = [l for l in layers if l[1] == "Softmax"]
    assert [p[0] for p in probs] == ["loss1/prob", "loss2/prob"], "the TEST net puts Softmax in front of the auxiliary Accuracy layers"
    bottoms = _bottoms(os.path.join(REF, "models/inception_v2/train_val.prototxt"))
    for name, _, shp in probs:
        assert shp == shapes[bottoms[name]] == (4, 1000), (name, shp)


@pytest.mark.parametrize("model,dims", [("bvlc_alexnet", (10, 1000)), ("bvlc_googlenet", (10, 1000)), ("bvlc_reference_caffenet", (10, 1000))])
def test_deploy_nets_end_in_prob(model, dims):
    n = _net(os.path.join(REF, "models", model, "deploy.prototxt"), "TEST")
    last = n.layers()[-1]
    assert last[0] == "prob" and last[1] == "Softmax" and last[2] == dims
    assert n.loss_blob() == ""
    assert not any(nb for nb, _ in n.backward_plan())                  # nothing reaches a loss


_IN = 'layer { name: "x" type: "Input" top: "x" top: "y" input_param { shape { dim: 2 dim: 3 dim: 4 dim: 5 } shape { dim: 2 dim: 7 } } }\n'


@pytest.mark.parametrize("bad,msg", [
    ('layer { name: "s" type: "Softmax" bottom: "x" top: "s" softmax_param { axis: 4 } }', r"axis 4 out of range for 4-D Blob with shape 2 3 4 5 \(120\)"),
    ('layer { name: "s" type: "Softmax" bottom: "x" top: "s" softmax_param { axis: -5 } }', r"axis -5 out of range for 4-D Blob"),
    ('layer { name: "f" type: "Flatten" bottom: "x" top: "f" flatten_param { axis: 7 } }', r"axis 7 out of range for 4-D Blob"),
    ('layer { name: "f" type: "Flatten" bottom: "x" top: "x" }', "Flatten Layer does not allow in-place computation."),
    ('layer { name: "l" type: "SigmoidCrossEntropyLoss" bottom: "x" bottom: "y" top: "l" }',
     "SIGMOID_CROSS_ENTROPY_LOSS layer inputs must have the same count."),
    ('layer { name: "l" type: "EuclideanLoss" bottom: "x" bottom: "y" top: "l" }', "Inputs must have the same dimension."),
])
def test_reference_shape_errors(bad, msg):
    from caffe_mpi_b200 import host_api as h
    with pytest.raises(h.HostError, match=msg):
        _net(_IN + bad, is_text=True)


def test_softmax_axis_and_flatten_shapes_in_the_graph():
    n = _net(_IN + 'layer { name: "s" type: "Softmax" bottom: "x" top: "s" softmax_param { axis: -1 } }\n'
                   'layer { name: "f" type: "Flatten" bottom: "s" top: "f" flatten_param { axis: 1 end_axis: 2 } }\n', is_text=True)
    shapes = {l[0]: l[2] for l in n.layers()}
    assert shapes["s"] == (2, 3, 4, 5) and shapes["f"] == (2, 12, 5)


def test_autoencoder_spec_renders_and_prunes():
    spec = nlo.autoencoder()
    n = _net(nlo.to_prototxt(spec), is_text=True)
    assert n.loss_blob() == "cross_entropy_loss"
    names = [l[0] for l in n.layers()]
    assert names.count("loss") == 2
    plan = n.backward_plan()
    assert plan[names.index("decode1neuron")][0] is False and plan[-1][0] is False
    assert [p[0] for p in n.learnable_params()] == [nm for nm, _, _ in nlo.param_shapes(spec)]


def test_force_backward_keeps_every_layer_but_the_label_bottoms():
    """net.cpp:342-360: with force_backward every layer runs backward, after pruning; a loss layer's label bottom still gets none."""
    text = nlo.to_prototxt(nlo.autoencoder())
    names = [l[0] for l in _net(text, is_text=True).layers()]
    forced = _net("force_backward: true\n" + text, is_text=True).backward_plan()
    assert forced[names.index("decode1neuron")] == (True, [True])
    assert forced[len(names) - 1] == (True, [True, True])               # EuclideanLoss: both bottoms
    assert forced[len(names) - 3] == (True, [True, False])              # SigmoidCrossEntropyLoss: never the target
    assert forced[0] == (False, [])                                     # the Input layer

"""Named parameter sharing, Slice and ContrastiveLoss without a GPU: the float64 ContrastiveLoss oracle against the closed forms of
the reference's test_contrastive_loss_layer.cpp and finite differences, Slice's shapes and error messages (test_slice_layer.cpp),
and the graph Net builds for the reference's MNIST siamese example: owners, multipliers, need-backward and the sharing refusals."""
import os
import re

import numpy as np
import pytest

import siamese_oracle as so
from caffe_mpi_b200 import host_api

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIAMESE = os.path.join(ROOT, "tests", "golden", "reference_models", "examples", "siamese")
TRAIN_TEST = os.path.join(SIAMESE, "mnist_siamese_train_test.prototxt")


# ------------------------------------------------------------------------------------------------------------ ContrastiveLoss oracle
def _pairs(seed, N=512, C=2):
    rng = np.random.default_rng(seed)      # the layer test's fillers: uniform [-1, 1] features, 0 / 1 labels
    return rng.uniform(-1, 1, (N, C)), rng.uniform(-1, 1, (N, C)), rng.integers(0, 2, N).astype(np.float64)


@pytest.mark.parametrize("legacy", [False, True], ids=["TestForward", "TestForwardLegacy"])
def test_contrastive_oracle_matches_layer_test_closed_form(legacy):
    a, b, y = _pairs(3)
    margin = 1.0
    loss = 0.0
    for i in range(len(a)):                 # test_contrastive_loss_layer.cpp's loops, term by term
        dist_sq = sum((a[i, j] - b[i, j]) ** 2 for j in range(a.shape[1]))
        if y[i]:
            loss += dist_sq
        elif legacy:
            loss += max(margin - dist_sq, 0.0)
        else:
            dist = max(margin - np.sqrt(dist_sq), 0.0)
            loss += dist * dist
    loss /= len(a) * 2.0
    got, _, _ = so.contrastive_forward(a, b, y, margin, legacy)
    assert abs(got - loss) <= 1e-12 * abs(loss)


@pytest.mark.parametrize("legacy", [False, True], ids=["new", "legacy"])
def test_contrastive_oracle_gradient_matches_finite_differences(legacy):
    a, b, y = _pairs(11, N=64, C=5)
    margin = 2.0 if not legacy else 4.0
    _, diff, d2 = so.contrastive_forward(a, b, y, margin, legacy)
    da, db = so.contrastive_backward(diff, d2, y, margin, legacy)
    keep = (np.sqrt(d2) > 0.05) & (np.abs(margin - (d2 if legacy else np.sqrt(d2))) > 1e-3)   # away from d = 0 and the hinge
    h = 1e-6
    for (X, G) in ((a, da), (b, db)):
        num = np.zeros_like(X)
        for i in range(X.shape[0]):
            for j in range(X.shape[1]):
                Xp, Xm = X.copy(), X.copy()
                Xp[i, j] += h
                Xm[i, j] -= h
                args_p = (Xp, b) if X is a else (a, Xp)
                args_m = (Xm, b) if X is a else (a, Xm)
                num[i, j] = (so.contrastive_forward(*args_p, y, margin, legacy)[0] - so.contrastive_forward(*args_m, y, margin, legacy)[0]) / (2 * h)
        # the analytic form divides by d + 1e-4 (the reference's), the derivative by d: relative 1e-4 / d apart
        tol = 1e-7 + np.abs(num) * (1e-4 / np.sqrt(d2)[:, None] + 1e-6)
        assert (np.abs(num - G) <= tol)[keep].all()


def test_contrastive_label_truncation():
    """static_cast<int>(y): 0.7 and -0.5 are dissimilar, 1.3 and -1 similar"""
    assert so.similar([0.0, 0.7, -0.5, 0.999, 1.0, 1.3, -1.0, 2.0]).tolist() == [False] * 4 + [True] * 4
    a = np.array([[0.3, 0.0]] * 4)
    b = np.zeros((4, 2))
    loss, _, d2 = so.contrastive_forward(a, b, np.array([0.7, 1.3, -0.5, -1.0]), margin=1.0)
    assert np.isclose(loss, ((1 - 0.3) ** 2 + 0.09 + (1 - 0.3) ** 2 + 0.09) / 8)


# ------------------------------------------------------------------------------------------------------------ Slice
def _slice_net(bottom_shape, tops, param):
    s = 'name: "s" layer { name: "in" type: "Input" top: "x" input_param { shape { %s } } }\n' % " ".join("dim: %d" % d for d in bottom_shape)
    s += 'layer { name: "slice" type: "Slice" bottom: "x" %s slice_param { %s } }\n' % (" ".join('top: "t%d"' % i for i in range(tops)), param)
    return s


def test_slice_setup_shapes():
    # test_slice_layer.cpp TestSetupNum / TestSetupChannels / TestTrivialSlice on a 6 x 12 x 2 x 3 bottom, then axis -1 and slice_dim
    got = _blob_shapes(_slice_net((6, 12, 2, 3), 3, "axis: 0"), ["t0", "t1", "t2"])
    assert got == [(2, 12, 2, 3)] * 3
    got = _blob_shapes(_slice_net((6, 12, 2, 3), 2, "slice_point: 3"), ["t0", "t1"])
    assert got == [(6, 3, 2, 3), (6, 9, 2, 3)]
    got = _blob_shapes(_slice_net((6, 12, 2, 3), 1, ""), ["t0"])
    assert got == [(6, 12, 2, 3)]
    got = _blob_shapes(_slice_net((6, 12, 2, 3), 3, "axis: -1 slice_point: 1 slice_point: 2"), ["t0", "t1", "t2"])
    assert got == [(6, 12, 2, 1)] * 3
    got = _blob_shapes(_slice_net((4, 2, 5, 5), 2, "slice_dim: 1 slice_point: 1"), ["t0", "t1"])
    assert got == [(4, 1, 5, 5)] * 2


def _blob_shapes(text, names):
    """the shapes of the tops `names`: Net's layer list reports each layer's first top, so one ReLU per top reports it"""
    n = host_api.Net(text + "".join('layer { name: "r%s" type: "ReLU" bottom: "%s" top: "r%s" }\n' % (t, t, t) for t in names),
                     "TRAIN", is_text=True)
    by_name = {nm: tuple(s) for nm, ty, s in n.layers()}
    return [by_name["r" + t] for t in names]


@pytest.mark.parametrize("param,tops,msg", [
    ("axis: 1 slice_dim: 1", 2, "Either axis or slice_dim should be specified; not both."),
    ("axis: 1 slice_point: 3 slice_point: 6", 2, "slice_point_.size() == top.size() - 1 (2 vs. 1)"),
    ("axis: 1 slice_point: 6 slice_point: 3", 3, "slice_point_[i] > prev (3 vs. 6)"),
    ("axis: 1", 5, "Number of top blobs (5) should evenly divide input slice axis (12)"),
    ("axis: 4", 2, "axis 4 out of range for 4-D Blob with shape 6 12 2 3 (432)"),
    ("slice_dim: 4", 2, "slice_dim out of range."),
    ("axis: 2 slice_point: 1 slice_point: 2", 3, "top.size() <= bottom_slice_axis (3 vs. 2)"),
    ("axis: 1 slice_point: 13", 2, "shape[i] >= 0 (-1 vs. 0)"),
])
def test_slice_reference_errors(param, tops, msg):
    with pytest.raises(host_api.HostError) as e:
        host_api.Net(_slice_net((6, 12, 2, 3), tops, param), "TRAIN", is_text=True)
    assert msg in str(e.value)


# ------------------------------------------------------------------------------------------------------------ the siamese nets
def _net(phase, text=None):
    if text is None:
        return host_api.Net(TRAIN_TEST, phase, default_channels=2, default_size=28)
    return host_api.Net(text, phase, is_text=True, default_channels=2, default_size=28)


OWNERS = ["conv1", "conv1", "conv2", "conv2", "ip1", "ip1", "ip2", "ip2", "feat", "feat"]


@pytest.mark.parametrize("phase", ["TRAIN", "TEST"])
def test_siamese_net_has_ten_owned_params(phase):
    n = _net(phase)
    lp = n.learnable_params()
    assert [p[0] for p in lp] == OWNERS
    assert [p[1] for p in lp] == [500, 20, 25000, 50, 400000, 500, 5000, 10, 20, 2]
    assert [p[2] for p in lp] == [1, 2] * 5 and all(p[3] == 1 for p in lp)
    np_ = n.net_params()
    assert len(np_) == 20
    assert [o for _, _, o, _ in np_] == [-1] * 10 + list(range(10))
    for i in range(10):                   # each _p layer's blob maps to its twin's learnable id
        assert np_[10 + i][0] == OWNERS[i] + "_p" and np_[10 + i][1] == np_[i][1] and np_[10 + i][3] == i


def test_siamese_need_backward_and_loss_blob():
    n = _net("TRAIN")
    assert n.loss_blob() == "loss"
    plan = dict(zip([l[0] for l in n.layers()], n.backward_plan()))
    assert plan["pair_data"] == (False, [])
    assert plan["slice_pair"] == (False, [False])          # the data needs no gradient
    assert plan["conv1"] == (True, [False]) and plan["conv1_p"] == (True, [False])
    assert plan["loss"] == (True, [True, True, False])     # never into the similarity label
    shapes = {nm: s for nm, _, s in n.layers()}
    assert shapes["slice_pair"] == (64, 1, 28, 28) and shapes["feat"] == (64, 2)


def test_siamese_without_names_lists_twenty_params():
    text = re.sub(r'\n\s*name: "\w+_[wb]"', "", open(TRAIN_TEST).read())
    n = _net("TRAIN", text)
    assert len(n.learnable_params()) == 20
    assert all(o == -1 for _, _, o, _ in n.net_params())


def test_siamese_force_backward_keeps_the_label_out():
    text = "force_backward: true\n" + open(TRAIN_TEST).read()
    plan = dict(zip([l[0] for l in _net("TRAIN", text).layers()], _net("TRAIN", text).backward_plan()))
    assert plan["loss"] == (True, [True, True, False])


def _two_ips(p1, p2, n1=4, n2=4):
    return ('name: "shared" layer { name: "in" type: "Input" top: "x" top: "t" input_param { shape { dim: 2 dim: 3 } '
            'shape { dim: 2 dim: %d } } }\n'
            'layer { name: "ip1" type: "InnerProduct" bottom: "x" top: "y1" %s inner_product_param { num_output: %d } }\n'
            'layer { name: "ip2" type: "InnerProduct" bottom: "x" top: "y2" %s inner_product_param { num_output: %d } }\n'
            'layer { name: "loss" type: "EuclideanLoss" bottom: "y1" bottom: "y2" top: "loss" }\n' % (n1, p1, n1, p2, n2))


def test_shape_mismatch_message():
    with pytest.raises(host_api.HostError) as e:
        _net("TRAIN", _two_ips('param { name: "w" }', 'param { name: "w" }', 4, 5))
    assert ("Cannot share param 'w' owned by layer 'ip1' with layer 'ip2'; shape mismatch.  Owner layer param shape is 4 3 (12); "
            "sharing layer expects shape 5 3 (15)") in str(e.value)


def test_lr_and_decay_mult_mismatch_messages():
    with pytest.raises(host_api.HostError) as e:
        _net("TRAIN", _two_ips('param { name: "w" lr_mult: 1 }', 'param { name: "w" lr_mult: 2 }'))
    assert "Shared param 'w' has mismatched lr_mult." in str(e.value)
    with pytest.raises(host_api.HostError) as e:
        _net("TRAIN", _two_ips('param { name: "w" decay_mult: 1 }', 'param { name: "w" decay_mult: 0 }'))
    assert "Shared param 'w' has mismatched decay_mult." in str(e.value)


def test_unset_owner_multiplier_adopts_the_sharers():
    n = _net("TRAIN", _two_ips('param { name: "w" } param { decay_mult: 0 }', 'param { name: "w" lr_mult: 3 decay_mult: 0.5 }'))
    lp = n.learnable_params()
    assert len(lp) == 3                                   # ip1 w (shared), ip1 b, ip2 b
    assert lp[0][0] == "ip1" and lp[0][2] == 3.0 and lp[0][3] == 0.5
    assert lp[1][3] == 0.0


def _permissive(b_bottom, b_out):
    return ('name: "p" layer { name: "in" type: "Input" top: "x" input_param { shape { dim: 2 dim: 6 } } }\n'
            'layer { name: "a" type: "InnerProduct" bottom: "x" top: "a" param { name: "w" } inner_product_param { num_output: 4 } }\n'
            'layer { name: "b" type: "InnerProduct" bottom: "%s" top: "b" param { name: "w" share_mode: PERMISSIVE } '
            'inner_product_param { num_output: %d } }\n' % (b_bottom, b_out))


def test_permissive_share_mode_with_other_shape_is_refused():
    with pytest.raises(host_api.HostError) as e:               # 2 x 6 against 4 x 6: the reference's count check
        _net("TRAIN", _permissive("x", 2))
    assert ("Cannot share param 'w' owned by layer 'a' with layer 'b'; count mismatch.  Owner layer param shape is 4 6 (24); "
            "sharing layer shape is 2 6 (12)") in str(e.value)
    with pytest.raises(host_api.HostError) as e:               # 6 x 4 against 4 x 6: the reference would reshape; not built
        _net("TRAIN", _permissive("a", 6))
    assert "share_mode PERMISSIVE with a different shape is not built" in str(e.value)
    assert len(_net("TRAIN", _permissive("x", 4)).learnable_params()) == 3   # the same shape: STRICT sharing


def test_batchnorm_statistics_cannot_be_shared():
    bn = ('layer { name: "%s" type: "BatchNorm" bottom: "x" top: "%s" param { name: "mean" lr_mult: 0 } param { lr_mult: 0 } '
          'param { lr_mult: 0 } }\n')
    head = 'name: "bn" layer { name: "in" type: "Input" top: "x" input_param { shape { dim: 2 dim: 3 dim: 4 dim: 4 } } }\n'
    _net("TRAIN", head + bn % ("bn1", "y1"))              # one named statistics blob alone is fine
    with pytest.raises(host_api.HostError) as e:
        _net("TRAIN", head + bn % ("bn1", "y1") + bn % ("bn2", "y2"))
    assert "two layers would update one running statistic" in str(e.value)

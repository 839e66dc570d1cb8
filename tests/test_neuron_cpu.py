"""The neuron layers without a device: the float64 forms of tests/neuron_oracle.py against the closed forms of the reference's
layer tests (test_neuron_layer.cpp, test_power_layer.cpp, test_threshold_layer.cpp) and against finite differences; Net's parsing,
shapes, PReLU's slope blob and the refusals with their messages; and b2c_debug_neuron_plan pinning each launch regime."""
import numpy as np
import pytest

import neuron_oracle as no
from caffe_mpi_b200 import capi, host_api

RNG = np.random.default_rng(11)
X = RNG.standard_normal((2, 3, 4, 5))                 # the reference tests' 2 x 3 x 4 x 5 Gaussian bottom


# ---- closed forms of the reference's layer tests ------------------------------------------------------------------------------
def test_absval_and_bnll():
    np.testing.assert_array_equal(no.forward("ABSVAL", X, {}), np.abs(X))
    y = no.forward("BNLL", X, {})
    assert (y >= 0).all() and (y >= X).all()                                   # TestBNLL: top >= 0 and top >= bottom
    np.testing.assert_allclose(y, np.log1p(np.exp(X)), rtol=1e-14)


@pytest.mark.parametrize("alpha", [0.5, 0.0])                                  # ELU, ELUasReLU
def test_elu(alpha):
    y = no.forward("ELU", X, {"alpha": alpha})
    want = np.where(X > 0, X, alpha * (np.exp(X) - 1))
    np.testing.assert_allclose(y, want, rtol=1e-12, atol=1e-15)
    if alpha == 0:
        np.testing.assert_array_equal(y, np.maximum(X, 0))


@pytest.mark.parametrize("base,scale,shift", [(-1, 1, 0), (2, 1, 0), (-1, 1, 1), (2, 1, 1), (2, 3, 0), (2, 3, 1), (-1, 3, 1), (0.5, 2, -1)])
def test_exp_and_log(base, scale, shift):
    """TestExpLayer / TestLogLayer: y = base^(shift + scale x) and y = log_base(shift + scale x) (base -1: e)"""
    q = {"base": base, "scale": scale, "shift": shift}
    b = np.e if base == -1 else base
    np.testing.assert_allclose(no.forward("EXP", X, q), np.exp(np.log(b) * (shift + scale * X)), rtol=1e-13)
    xp = np.abs(X) + 0.5                                                        # a positive argument, as the log test draws
    arg = shift + scale * xp
    ok = arg > 0
    np.testing.assert_allclose(no.forward("LOG", xp, q)[ok], (np.log(arg) / np.log(b))[ok], rtol=1e-13)
    inner, outer = no.exp_constants(base, scale, shift)
    assert np.isclose(inner, np.log(b) * scale, rtol=1e-6) and np.isclose(outer, b ** shift, rtol=1e-6)
    bs, bns = no.log_constants(base, scale)
    assert np.isclose(bs, 1 / np.log(b), rtol=1e-6) and np.isclose(bns, scale / np.log(b), rtol=1e-6)


@pytest.mark.parametrize("power,scale,shift", [(0.37, 0.83, -2.4), (0.37, 0.83, 0.0), (0.0, 0.83, -2.4), (1.0, 0.83, -2.4),
                                               (2.0, 0.34, -2.4), (2.0, 0.5, 0.0), (2.0, 0.0, 1.5), (-1.5, 0.8, 0.0)])
def test_power(power, scale, shift):
    """TestPowerLayer: y = (shift + scale x)^power, NaN where a negative base meets a non-integer power; power 0 or scale 0: the
    constant"""
    q = {"power": power, "scale": scale, "shift": shift}
    with np.errstate(invalid="ignore", divide="ignore"):
        y = no.forward("POWER", X, q)
        want = np.full_like(X, 1.0 if power == 0 else shift ** power) if power * scale == 0 else np.power(shift + scale * X, power)
    np.testing.assert_array_equal(np.isnan(y), np.isnan(want))
    ok = ~np.isnan(want)
    np.testing.assert_allclose(y[ok], want[ok], rtol=1e-14)


@pytest.mark.parametrize("threshold", [0.0, 0.5, -0.2])
def test_threshold(threshold):
    y = no.forward("THRESHOLD", X, {"threshold": threshold})
    assert set(np.unique(y)) <= {0.0, 1.0}
    np.testing.assert_array_equal(y, (X > threshold).astype(np.float64))


@pytest.mark.parametrize("shared", [False, True])
def test_prelu_forward_and_consistency_with_relu(shared):
    slope = np.array([0.25]) if shared else RNG.uniform(0.1, 0.9, 3)
    y = no.prelu_forward(X, slope, shared)
    s = np.full(3, slope[0]) if shared else slope
    for c in range(3):
        xc = X[:, c]
        np.testing.assert_array_equal(y[:, c], np.where(xc > 0, xc, xc * s[c]))
    np.testing.assert_array_equal(no.prelu_forward(X, np.zeros(1 if shared else 3), shared), np.maximum(X, 0))   # ConsistencyReLU
    dy = RNG.standard_normal(X.shape)
    dx, _, _ = no.prelu_backward(X, dy, np.zeros(1 if shared else 3), shared)
    np.testing.assert_array_equal(dx, dy * (X > 0))


# ---- finite differences ------------------------------------------------------------------------------------------------------
FD_CASES = [("ELU", {"alpha": 0.5}), ("ELU", {"alpha": 0.0}), ("ABSVAL", {}), ("BNLL", {}), ("EXP", {"base": 2, "scale": 3, "shift": 1}),
            ("EXP", {}), ("LOG", {"base": 2, "scale": 3, "shift": 1}), ("LOG", {}), ("POWER", {"power": 0.37, "scale": 0.83, "shift": 2.4}),
            ("POWER", {"power": 0.37, "scale": 0.83, "shift": 0.0}), ("POWER", {"power": 2.0, "scale": 0.34, "shift": -2.4}),
            ("POWER", {"power": 1.0, "scale": 0.83, "shift": -2.4}), ("POWER", {"power": 0.0, "scale": 0.83, "shift": -2.4})]


@pytest.mark.parametrize("case", range(len(FD_CASES)))
def test_gradient_against_finite_differences(case):
    kind, q = FD_CASES[case]
    x = RNG.standard_normal(200)
    x = x[np.abs(x) > 1e-2]                                                     # away from the kinks of ELU / AbsVal
    if kind in ("LOG", "POWER"):
        x = np.abs(x) + 0.2                                                     # inside the domain
    dy = RNG.standard_normal(x.shape)
    h = 1e-6
    fd = dy * (no.forward(kind, x + h, q) - no.forward(kind, x - h, q)) / (2 * h)
    np.testing.assert_allclose(no.backward(kind, x, dy, q), fd, rtol=1e-6, atol=1e-7)


@pytest.mark.parametrize("shared", [False, True])
def test_prelu_gradient_against_finite_differences(shared):
    x = X.copy()
    x[np.abs(x) < 1e-2] = 0.5
    slope = np.array([0.3]) if shared else RNG.uniform(0.1, 0.9, 3)
    dy = RNG.standard_normal(x.shape)
    dx, ds, _ = no.prelu_backward(x, dy, slope, shared)
    h = 1e-6
    for k in range(slope.size):
        sp, sm = slope.copy(), slope.copy()
        sp[k] += h
        sm[k] -= h
        fd = (dy * (no.prelu_forward(x, sp, shared) - no.prelu_forward(x, sm, shared))).sum() / (2 * h)
        assert abs(ds[k] - fd) <= 1e-6 * max(1, abs(fd))
    fdx = dy * (no.prelu_forward(x + h, slope, shared) - no.prelu_forward(x - h, slope, shared)) / (2 * h)
    np.testing.assert_allclose(dx, fdx, rtol=1e-6, atol=1e-8)


# ---- Net: parsing, shapes, the slope blob, refusals ---------------------------------------------------------------------------
HEAD = ('name: "n" layer { name: "in" type: "Input" top: "data" top: "label" input_param { shape { dim: 2 dim: 4 dim: 3 dim: 3 } '
        'shape { dim: 2 } } }\n')
TAIL = ('layer { name: "ip" type: "InnerProduct" bottom: "%s" top: "ip" inner_product_param { num_output: 3 } }\n'
        'layer { name: "loss" type: "SoftmaxWithLoss" bottom: "ip" bottom: "label" top: "loss" }\n')


def net(layer, top="x"):
    return HEAD + layer + "\n" + TAIL % top


@pytest.mark.parametrize("ty,param", [("ELU", "elu_param { alpha: 0.5 }"), ("Power", "power_param { power: 2 }"), ("AbsVal", ""),
                                      ("BNLL", ""), ("Exp", "exp_param { base: 2 }"), ("Log", "log_param { shift: 1 }"),
                                      ("Threshold", "threshold_param { threshold: 0.1 }"), ("PReLU", "")])
def test_top_shapes_and_need_backward(ty, param):
    n = host_api.Net(net(f'layer {{ name: "x" type: "{ty}" bottom: "data" top: "x" {param} }}'), is_text=True)
    assert n.top_shape(1, 0) == (2, 4, 3, 3)
    assert n.backward_plan()[1][0] == (ty == "PReLU")            # only PReLU owns a parameter: the data needs no gradient
    c = ('layer { name: "c" type: "Convolution" bottom: "data" top: "c" convolution_param { num_output: 4 kernel_size: 1 } }\n'
         f'layer {{ name: "x" type: "{ty}" bottom: "c" top: "x" {param} }}')
    plan = host_api.Net(net(c), is_text=True).backward_plan()
    assert plan[2] == (True, [True])


@pytest.mark.parametrize("shared", [False, True])
def test_prelu_slope_blob(shared):
    layer = 'layer { name: "x" type: "PReLU" bottom: "data" top: "x" %s }' % ("prelu_param { channel_shared: true }" if shared else "")
    params = host_api.Net(net(layer), is_text=True).learnable_params()
    assert [p[:2] for p in params] == [("x", 1 if shared else 4), ("ip", 3 * 36), ("ip", 3)]
    lr = ('layer { name: "x" type: "PReLU" bottom: "data" top: "x" param { lr_mult: 2 decay_mult: 0 } }')
    assert host_api.Net(net(lr), is_text=True).learnable_params()[0][1:] == (4, 2.0, 0.0)


def test_prelu_slope_is_shared_by_name():
    two = ('layer { name: "a" type: "PReLU" bottom: "data" top: "a" param { name: "s" } }\n'
           'layer { name: "x" type: "PReLU" bottom: "a" top: "x" param { name: "s" } }')
    n = host_api.Net(net(two), is_text=True)
    assert [p[:2] for p in n.learnable_params()] == [("a", 4), ("ip", 3 * 36), ("ip", 3)]
    assert [(p[0], p[2]) for p in n.net_params()][:2] == [("a", -1), ("x", 0)]


REFUSED = {
    "exp_base": ('layer { name: "x" type: "Exp" bottom: "data" top: "x" exp_param { base: -2 } }', "base must be strictly positive."),
    "log_base": ('layer { name: "x" type: "Log" bottom: "data" top: "x" log_param { base: 0 } }', "base must be strictly positive."),
}


@pytest.mark.parametrize("case", ["exp_base", "log_base"])
def test_net_refusals(case):
    layer, msg = REFUSED[case]
    with pytest.raises(host_api.HostError, match=msg.replace(".", r"\.")):
        host_api.Net(net(layer), is_text=True)


def test_prelu_refuses_a_bottom_with_fewer_than_two_axes():
    bad = ('name: "n" layer { name: "in" type: "Input" top: "data" input_param { shape { dim: 6 } } }\n'
           'layer { name: "x" type: "PReLU" bottom: "data" top: "x" }\n')
    with pytest.raises(host_api.HostError, match=r"Number of axes of bottom blob must be >=2\."):
        host_api.Net(bad, is_text=True)


def test_tanh_and_scale_still_parse():
    for layer in ('layer { name: "x" type: "TanH" bottom: "data" top: "x" }', 'layer { name: "x" type: "Scale" bottom: "data" top: "x" }'):
        host_api.Net(net(layer), is_text=True)


# ---- the plan query -----------------------------------------------------------------------------------------------------------
def test_prelu_plan_regimes():
    stem = capi.neuron_plan("prelu_backward", 64, 64, 112 * 112)             # small C, large maps: several CTAs per channel
    assert stem["vec"] and stem["blocks_per_channel"] == 17 and stem["channels"] == 64 and stem["ctas"] == 17 * 64
    assert stem["workspace"] == 64 * 4 + 64 * 17 * 4
    deep = capi.neuron_plan("prelu_backward", 64, 2048, 7 * 7)               # large C, 7 x 7: one CTA per channel, no workspace
    assert not deep["vec"] and deep["blocks_per_channel"] == 1 and deep["ctas"] == 2048 and deep["workspace"] == 0
    assert deep["stripe"] == 13                                               # 3136 values over 256 threads
    shared = capi.neuron_plan("prelu_backward", 64, 64, 112 * 112, shared=True)
    assert shared["channels"] == 1 and shared["blocks_per_channel"] == 1056 and shared["vec"]
    tiny = capi.neuron_plan("prelu_backward", 2, 3, 1)
    assert tiny == dict(vec=False, ctas=3, threads=256, blocks_per_channel=1, stripe=1, channels=3, workspace=0)
    assert capi.neuron_plan("prelu_backward", 2, 3, 4)["vec"]
    assert not capi.neuron_plan("prelu_backward", 2, 3, 4, ptrs=(4, 0, 0))["vec"]   # a misaligned pointer: one float at a time
    fwd = capi.neuron_plan("prelu_forward", 64, 64, 112 * 112)
    assert fwd["ctas"] == stem["ctas"] and fwd["workspace"] == 0
    for N, Cc, dim, sh in ((64, 64, 112 * 112, False), (1, 1, 1, False), (3, 7, 5, True)):
        ws = capi.prelu_workspace_bytes(N, Cc, dim, sh)
        assert ws == capi.neuron_plan("prelu_backward", N, Cc, dim, shared=sh)["workspace"]


def test_elementwise_plan():
    p = capi.neuron_plan("forward", 1 << 20, kind="EXP")
    assert p["vec"] and p["threads"] == 256 and p["ctas"] >= 1
    assert not capi.neuron_plan("backward", 1000, kind="LOG", ptrs=(0, 0, 8, 4))["vec"]
    assert capi.neuron_plan("forward", 0, kind="ELU")["ctas"] == 0


@pytest.mark.parametrize("args", [("prelu_backward", 0, 3, 4), ("prelu_forward", 2, 0, 4), ("prelu_backward", 2, 3, 0),
                                  ("prelu_backward", 1 << 16, 1, 1 << 15), ("prelu_forward", 1 << 12, 1 << 10, 1 << 10, True)])
def test_plan_refuses_bad_shapes(args):
    with pytest.raises(capi.B2CError, match="must be >= 1|2\\^31"):
        capi.neuron_plan(*args)


def test_plan_refuses_bad_op_and_kind():
    with pytest.raises(capi.B2CError, match="Threshold has no backward"):
        capi.neuron_plan("backward", 10, kind="THRESHOLD")
    out = (capi.C.c_int * 7)()
    with pytest.raises(capi.B2CError, match="op is"):
        capi.check(capi.lib().b2c_debug_neuron_plan(7, 0, 1, 1, 1, 0, None, 0, out, 7))
    with pytest.raises(capi.B2CError, match="unknown kind"):
        capi.check(capi.lib().b2c_debug_neuron_plan(0, 9, 1, 1, 1, 0, None, 0, out, 7))
    with pytest.raises(capi.B2CError, match="needs out"):
        capi.check(capi.lib().b2c_debug_neuron_plan(0, 0, 1, 1, 1, 0, None, 0, out, 6))


@pytest.mark.parametrize("N,Cc,dim,shared", [(32, 64, 32 * 32, True), (64, 64, 112 * 112, False), (16, 3, 15 * 15, False), (7, 2, 4099, False),
                                             (5, 3, 1000, True)])
def test_prelu_workspace_does_not_depend_on_alignment(N, Cc, dim, shared):
    """b2c_prelu_workspace_bytes takes no pointers: a call 4 bytes off (the scalar path) must fit in what it reports, so the
    CTAs per channel, and with them the workspace, come from the shape alone"""
    aligned = capi.neuron_plan("prelu_backward", N, Cc, dim, shared=shared)
    off = capi.neuron_plan("prelu_backward", N, Cc, dim, shared=shared, ptrs=(4, 0, 0))
    assert not off["vec"]
    assert off["blocks_per_channel"] == aligned["blocks_per_channel"] and off["ctas"] == aligned["ctas"]
    assert off["workspace"] == aligned["workspace"] == capi.prelu_workspace_bytes(N, Cc, dim, shared)

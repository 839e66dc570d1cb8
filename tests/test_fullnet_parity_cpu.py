"""The layer-by-layer checker of tests/test_fullnet_parity_gpu.py (tests/fullnet_walker.py) validated without a GPU: fed the
net oracle's own blobs, diffs and gradients (tests/netoracle.py) for the mini ResNet and the mini Inception net, it must find
them right to float32 rounding, and it must notice a wrong value of each kind.  Its float64 convolution must agree with the
checker library's float64-accumulating one."""
import numpy as np
import pytest

import oracle
import netoracle as no
import fullnet_walker as fw


def oracle_state(spec, rng, seed=1701):
    shapes = no.param_shapes(spec)
    params = []
    for _, kind, shp in shapes:
        if kind == "w":
            params.append((rng.standard_normal(shp) * np.sqrt(2.0 / np.prod(shp[1:]))).astype(np.float32))
        elif kind == "scale":
            params.append(rng.uniform(0.5, 1.5, shp).astype(np.float32))
        else:
            params.append(rng.uniform(-0.2, 0.2, shp).astype(np.float32))
    dshape = spec[0]["shape"]
    data = rng.standard_normal(dshape).astype(np.float32)
    label = rng.integers(0, 10, dshape[0]).astype(np.float32)
    _, grads, v, d = no.forward_backward(spec, params, data, label, seed=seed)
    per_layer = {}
    for (layer, _, _), p, g in zip(shapes, params, grads):
        per_layer.setdefault(layer, []).append((p.reshape(-1), np.asarray(g, np.float32).reshape(-1)))

    def fetch(name, diff):
        src = d if diff else v
        return np.asarray(src[name], np.float32).reshape(-1).copy()

    return fetch, per_layer, data, label


@pytest.mark.parametrize("net", ["mini_resnet", "mini_inception"])
def test_walker_reproduces_the_net_oracle(net, rng):
    spec = getattr(no, net)()
    layers = fw.parse_layers(no.to_prototxt(spec))
    assert [L["name"] for L in layers][1:] == [L["n"] for L in spec][1:]
    fetch, params, data, label = oracle_state(spec, rng)
    shapes = {}
    checks = fw.walk(layers, fetch, params, data.shape, label, shapes=shapes)
    bad = [c for c in checks if not (np.isfinite(c.err) and c.err <= (0.0 if c.bar == 0 else 1e-5))]
    assert not bad, bad
    # a forward-only re-walk on the stored shapes recomputes only the kinds asked for, with the same results
    again = fw.walk(layers, fetch, params, data.shape, label, forward_only=True, kinds={"Convolution"}, shapes=shapes)
    assert [c for c in again if c.what == "y"] == [c for c in checks if c.kind == "Convolution" and c.what == "y"]
    got = {(c.kind, c.what if not c.what.startswith("dx:") else "dx") for c in checks}
    # every check the GPU file relies on ran at least once on these nets
    want = {("Convolution", "y"), ("Convolution", "dW"), ("MAX", "y"), ("AVE", "y"), ("InnerProduct", "y"), ("InnerProduct", "dW"), ("InnerProduct", "db"),
            ("SoftmaxWithLoss", "loss"), ("ReLU", "mask_fwd"), ("ReLU", "mask_bwd")}
    if net == "mini_resnet":
        want |= {("Eltwise", "y"), ("Eltwise", "dx"), ("BatchNorm", "y"), ("BatchNorm", "dgamma"), ("BatchNorm", "dbeta")}
    else:
        want |= {("LRN", "y"), ("Concat", "y"), ("Concat", "dx"), ("Dropout", "mask_fwd"), ("Dropout", "mask_bwd"), ("Convolution", "db")}
    assert want <= got, want - got
    # the blob diffs of every consumer mix were checked: the net's every non-input blob but the loss tops has one
    diffed = {c.what[3:] for c in checks if c.what.startswith("dx:")}
    produced = {L["top"][0] for L in layers[1:] if L["type"] not in ("ReLU", "Dropout", "SoftmaxWithLoss")}
    assert diffed == produced


EXPECT = {"conv_y": {("inc/3x3", "y")}, "bn_dgamma": {("resA.1.conv2/bn", "dgamma")}, "concat_dx": {("inc/5x5", "dx:inc/5x5")},
          "relu_mask": {("inc/relu_1x1", "mask_bwd")}, "dropout_mask": {("aux/drop", "mask_fwd"), ("drop5", "mask_fwd")},
          "loss": {("aux/loss", "loss")}, "eltwise_y": {("resA.2.sum", "y")}}


@pytest.mark.parametrize("what", sorted(EXPECT))
def test_walker_flags_a_wrong_value(what, rng):
    """one element wrong, or one dropout stream off by an iteration: the walker reports that layer and tensor"""
    net = "mini_resnet" if what in ("eltwise_y",) else "mini_inception"
    spec = getattr(no, net)()
    layers = fw.parse_layers(no.to_prototxt(spec))
    fetch, params, data, label = oracle_state(spec, rng)
    iteration = 0
    blob, diff = None, False
    if what == "conv_y":
        blob = "inc/3x3"
    elif what == "concat_dx":
        blob, diff = "inc/5x5", True
    elif what == "relu_mask":
        blob, diff = "inc/1x1", True
    elif what == "eltwise_y":
        blob = "resA.2.sum"
    elif what == "loss":
        blob = "aux/loss1"
    elif what == "bn_dgamma":
        pass
    elif what == "dropout_mask":
        iteration = 1

    def bad_fetch(name, d):
        a = fetch(name, d)
        if name == blob and d == diff:
            if what == "relu_mask":                          # a gradient leaks through a position the ReLU cut
                k = int(np.flatnonzero(fetch(name, False) <= 0)[0])
                a[k] = 1e-3
            else:
                k = int(np.argmax(np.abs(a)))
                a[k] = a[k] * (1 + 1e-3) if what != "eltwise_y" else np.nextafter(a[k], np.float32(np.inf))
        return a

    if what == "bn_dgamma":
        spec = no.mini_resnet()
        layers = fw.parse_layers(no.to_prototxt(spec))
        fetch, params, data, label = oracle_state(spec, rng)
        g = params["resA.1.conv2/bn"][0][1].copy()
        g[0] *= 1.01
        params["resA.1.conv2/bn"][0] = (params["resA.1.conv2/bn"][0][0], g)
        bad_fetch = fetch
    checks = fw.walk(layers, bad_fetch, params, data.shape, label, iteration=iteration)
    bad = {(c.layer, c.what) for c in fw.failures(checks)}
    assert EXPECT[what] <= bad, (what, sorted(bad))


@pytest.mark.parametrize("shape", [(2, 8, 9, 9, 16, 3, 1, 1, 1), (2, 6, 11, 11, 8, 5, 2, 2, 2), (1, 32, 7, 7, 64, 1, 1, 0, 1),
                                   (2, 3, 15, 15, 8, 7, 2, 3, 1)])
def test_float64_conv_matches_the_checker_library(shape, rng):
    N, C, H, W, O, k, s, p, g = shape
    prm = oracle.ConvParams.make(N, C, H, W, O, k, s, p, 1, g, True)
    x = rng.standard_normal(prm.x_shape()).astype(np.float32)
    w = rng.standard_normal(prm.w_shape()).astype(np.float32)
    b = rng.standard_normal(O).astype(np.float32)
    dy = rng.standard_normal(prm.y_shape()).astype(np.float32)
    y = fw.conv_forward(x, w, b, s, p, g)
    ref = np.asarray(oracle.conv_forward(prm, x, w, b, acc64=True), np.float64).reshape(y.shape)
    assert fw.rel(y, ref) <= 1e-6
    dw, db, dx = fw.conv_backward(x, w, dy, s, p, g)
    dw_r, db_r, dx_r = oracle.conv_backward(prm, x, w, dy, acc64=True)
    assert fw.rel(dw, np.asarray(dw_r).reshape(dw.shape)) <= 1e-6
    assert fw.rel(db, np.asarray(db_r)) <= 1e-6
    assert fw.rel(dx, np.asarray(dx_r).reshape(dx.shape)) <= 1e-6


def test_pool_and_lrn_forms_match_the_layer_oracle(rng):
    """the vectorised float64 pooling / LRN forms against oracle/layers_oracle.py (ceil-mode windows, padding, first maximum)"""
    x = rng.standard_normal((2, 5, 13, 13)).astype(np.float32)
    x[0, 0, :4, :4] = 0                                   # ties: the first maximum wins
    for k, s, p in ((3, 2, 0), (3, 1, 1), (2, 2, 0), (5, 3, 0), (7, 1, 0)):
        y, arg = fw.max_pool_forward(x, k, s, p)
        ry, rm = lo_pool(x, 0, k, s, p)
        assert np.array_equal(y, ry) and np.array_equal(arg, rm), (k, s, p)
        dy = rng.standard_normal(y.shape).astype(np.float32)
        assert fw.rel(fw.max_pool_backward(dy, arg, x.shape), oracle.layers_oracle.pool_backward(dy, rm, x.shape, 0, (k, k), (s, s), (p, p))) <= 1e-6
        ya = fw.ave_pool_forward(x, k, s, p)
        assert fw.rel(ya, lo_pool(x, 1, k, s, p)[0]) <= 1e-6
        assert fw.rel(fw.ave_pool_backward(dy, x.shape, k, s, p),
                      oracle.layers_oracle.pool_backward(dy, None, x.shape, 1, (k, k), (s, s), (p, p))) <= 1e-6
    y, scale = fw.lrn_forward(x, 5, 1e-2, 0.75, 1.0)
    ry, rs = oracle.layers_oracle.lrn_forward(x, 5, 1e-2, 0.75, 1.0)
    assert fw.rel(y, ry) <= 1e-6 and fw.rel(scale, rs) <= 1e-6
    dy = rng.standard_normal(x.shape).astype(np.float32)
    assert fw.rel(fw.lrn_backward(x, y, scale, dy, 5, 1e-2, 0.75), oracle.layers_oracle.lrn_backward(x, ry, rs, dy, 5, 1e-2, 0.75)) <= 1e-5


def lo_pool(x, method, k, s, p):
    return oracle.layers_oracle.pool_forward(x, method, (k, k), (s, s), (p, p))

"""Float64 forms of the Softmax, Sigmoid, Flatten, SigmoidCrossEntropyLoss and EuclideanLoss layers, and a whole-net oracle for
the small nets built from them (an autoencoder-shaped MLP, a conv net ending in Softmax).  The per-layer forms restate the
reference's CPU code (softmax_layer.cpp, sigmoid_layer.cpp, sigmoid_cross_entropy_loss_layer.cpp, euclidean_loss_layer.cpp,
flatten_layer.cpp).  TEST INFRASTRUCTURE ONLY."""
import numpy as np
from oracle import layers_oracle as lo


def _view(x, axis):
    s = x.shape
    axis = axis + len(s) if axis < 0 else axis
    return x.reshape(int(np.prod(s[:axis], dtype=np.int64)), s[axis], int(np.prod(s[axis + 1:], dtype=np.int64))), axis


def softmax_forward(x, axis=1):
    """softmax over `axis`: max-shifted exp, divided by the channel sum (softmax_layer.cpp:24-60)."""
    v, _ = _view(np.asarray(x, np.float64), axis)
    e = np.exp(v - v.max(axis=1, keepdims=True))
    return (e / e.sum(axis=1, keepdims=True)).reshape(np.shape(x))


def softmax_backward(y, dy, axis=1):
    """dx = (dy - sum_c dy * y) * y (softmax_layer.cpp:63-90)."""
    yv, _ = _view(np.asarray(y, np.float64), axis)
    dv, _ = _view(np.asarray(dy, np.float64), axis)
    return ((dv - (dv * yv).sum(axis=1, keepdims=True)) * yv).reshape(np.shape(y))


def sigmoid_forward(x):
    return 1.0 / (1.0 + np.exp(-np.asarray(x, np.float64)))


def sigmoid_backward(y, dy):
    y = np.asarray(y, np.float64)
    return np.asarray(dy, np.float64) * y * (1.0 - y)


def sigmoid_ce_terms(x, t):
    """The reference's stable per-element expression, x (t - [x >= 0]) - log(1 + exp(x - 2 x [x >= 0]))."""
    x, t = np.asarray(x, np.float64), np.asarray(t, np.float64)
    pos = (x >= 0).astype(np.float64)
    return x * (t - pos) - np.log1p(np.exp(x - 2.0 * x * pos))


def sigmoid_ce_loss(x, t):
    """-sum(terms) / num (sigmoid_cross_entropy_loss_layer.cpp:35-45); num = the bottom's first axis."""
    return float(-sigmoid_ce_terms(x, t).sum() / np.shape(x)[0])


def sigmoid_ce_backward(x, t, loss_weight=1.0):
    return (sigmoid_forward(x) - np.asarray(t, np.float64)) * (loss_weight / np.shape(x)[0])


def euclidean_loss(a, b):
    d = np.asarray(a, np.float64) - np.asarray(b, np.float64)
    return float((d * d).sum() / np.shape(a)[0] / 2.0), d


def euclidean_backward(diff, num, loss_weight=1.0):
    """(gradient to bottom 0, gradient to bottom 1): +-loss_weight / num * diff (euclidean_loss_layer.cpp:25-38)."""
    g = diff * (loss_weight / num)
    return g, -g


def flatten_shape(shape, axis=1, end_axis=-1):
    n = len(shape)
    a, e = axis + n if axis < 0 else axis, end_axis + n if end_axis < 0 else end_axis
    return tuple(shape[:a]) + (int(np.prod(shape[a:e + 1], dtype=np.int64)),) + tuple(shape[e + 1:])


# ---- whole nets ---------------------------------------------------------------------------------------------------------
def autoencoder(batch=8, side=6, widths=(20, 10, 4), wd_branch=True):
    """mnist_autoencoder.prototxt in miniature: a Flatten target, an IP -> Sigmoid encoder and decoder (the code layer has no
    sigmoid), SigmoidCrossEntropyLoss on the decoder's logits, and a loss_weight 0 Sigmoid -> EuclideanLoss branch.  Two layers
    are named `loss`, as in the reference file."""
    d = side * side
    spec = [dict(t="data", shape=(batch, 1, side, side)), dict(t="flatten", n="flatdata", b="data")]
    src, k = "data", 0
    enc = list(widths)
    dec = list(reversed(widths[:-1])) + [d]
    for i, w in enumerate(enc):
        n = f"encode{i + 1}"
        spec.append(dict(t="fc", n=n, b=src, o=w))
        src = n
        if i + 1 < len(enc):
            spec.append(dict(t="sigmoid", n=n + "neuron", b=n))
            src = n + "neuron"
    for i, w in enumerate(dec):
        n = f"decode{len(dec) - i}"
        spec.append(dict(t="fc", n=n, b=src, o=w))
        src = n
        if i + 1 < len(dec):
            spec.append(dict(t="sigmoid", n=n + "neuron", b=n))
            src = n + "neuron"
    spec.append(dict(t="sigce", n="loss", b=[src, "flatdata"], top="cross_entropy_loss", w=1.0))
    if wd_branch:
        spec += [dict(t="sigmoid", n=src + "neuron", b=src), dict(t="euclid", n="loss", b=[src + "neuron", "flatdata"], top="l2_error", w=0.0)]
    return spec


def to_prototxt(spec):
    s = 'name: "mini_autoencoder"\n'
    for L in spec:
        t = L["t"]
        if t == "data":
            N, Cc, H, W = L["shape"]
            s += f'layer {{ name: "data" type: "Input" top: "data" input_param {{ shape {{ dim: {N} dim: {Cc} dim: {H} dim: {W} }} }} }}\n'
        elif t == "flatten":
            s += f'layer {{ name: "{L["n"]}" type: "Flatten" bottom: "{L["b"]}" top: "{L["n"]}" }}\n'
        elif t == "fc":
            s += (f'layer {{ name: "{L["n"]}" type: "InnerProduct" bottom: "{L["b"]}" top: "{L["n"]}" param {{ lr_mult: 1 decay_mult: 1 }} '
                  f'param {{ lr_mult: 1 decay_mult: 0 }} inner_product_param {{ num_output: {L["o"]} weight_filler {{ type: "gaussian" std: 0.1 }} '
                  f'bias_filler {{ type: "constant" value: 0 }} }} }}\n')
        elif t == "sigmoid":
            s += f'layer {{ name: "{L["n"]}" type: "Sigmoid" bottom: "{L["b"]}" top: "{L["n"]}" }}\n'
        elif t in ("sigce", "euclid"):
            ty = "SigmoidCrossEntropyLoss" if t == "sigce" else "EuclideanLoss"
            s += (f'layer {{ name: "{L["n"]}" type: "{ty}" bottom: "{L["b"][0]}" bottom: "{L["b"][1]}" top: "{L["top"]}" '
                  f'loss_weight: {L["w"]} }}\n')
    return s


def param_shapes(spec):
    shapes, dims = [], {}
    for L in spec:
        if L["t"] == "data":
            dims["data"] = int(np.prod(L["shape"][1:]))
        elif L["t"] == "fc":
            shapes += [(L["n"], "w", (L["o"], dims[L["b"]])), (L["n"], "b", (L["o"],))]
            dims[L["n"]] = L["o"]
        elif L["t"] in ("sigmoid", "flatten"):
            dims[L["n"]] = dims[L["b"]]
    return shapes


def forward_backward(spec, params, data):
    """(reported loss = cross_entropy_loss, grads in param_shapes order, forward values).  The weight-0 branch runs forward only."""
    N = data.shape[0]
    v = {"data": np.asarray(data, np.float64), "flatdata": np.asarray(data, np.float64).reshape(N, -1)}
    pidx, pi = {}, 0
    for L in spec:
        t = L["t"]
        if t == "fc":
            pidx[L["n"]] = pi
            pi += 2
            v[L["n"]] = lo.ip_forward(v[L["b"]].reshape(N, -1), params[pidx[L["n"]]], params[pidx[L["n"]] + 1]).astype(np.float64)
        elif t == "sigmoid":
            v[L["n"]] = sigmoid_forward(v[L["b"]])
        elif t == "sigce":
            v[L["top"]] = sigce = sigmoid_ce_loss(v[L["b"][0]], v[L["b"][1]])
        elif t == "euclid":
            v[L["top"]] = euclidean_loss(v[L["b"][0]], v[L["b"][1]])[0]
    grads = [np.zeros_like(p, dtype=np.float64) for p in params]
    d = {}
    for L in reversed(spec):
        t = L["t"]
        if t == "sigce":
            d[L["b"][0]] = sigmoid_ce_backward(v[L["b"][0]], v[L["b"][1]], L["w"])
        elif t == "sigmoid" and L["n"] in d:
            d[L["b"]] = sigmoid_backward(v[L["n"]], d[L["n"]])
        elif t == "fc" and L["n"] in d:
            x = v[L["b"]].reshape(N, -1)
            w = np.asarray(params[pidx[L["n"]]], np.float64)
            grads[pidx[L["n"]]] = d[L["n"]].T @ x
            grads[pidx[L["n"]] + 1] = d[L["n"]].sum(axis=0)
            if L["b"] != "data":
                d[L["b"]] = d[L["n"]] @ w
    return sigce, grads, v

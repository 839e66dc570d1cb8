"""Float64 forms of the neuron layers (elu, power, absval, bnll, exp, log, threshold and prelu _layer.cpp), float32 restatements of
the rules the kernels compute exactly, the constants each LayerSetUp derives, and a float64 net oracle (torch, CPU) for the
small neuron net the GPU suite trains through TrainNet."""
import numpy as np

KINDS = ("ELU", "POWER", "ABSVAL", "BNLL", "EXP", "LOG", "THRESHOLD")
f32 = np.float32


# ---- the derived constants, as the reference's LayerSetUp computes them in float -----------------------------------------------
def exp_constants(base=-1.0, scale=1.0, shift=0.0):
    """(inner_scale, outer_scale) of exp_layer.cpp:9-29."""
    base, scale, shift = f32(base), f32(scale), f32(shift)
    log_base = f32(1) if base == -1 else f32(np.log(base))
    inner = f32(log_base * scale)
    outer = f32(1) if shift == 0 else (f32(np.power(base, shift)) if base != -1 else f32(np.exp(shift)))
    return float(inner), float(outer)


def log_constants(base=-1.0, scale=1.0):
    """(base_scale, backward_num_scale) of log_layer.cpp:9-35."""
    base, scale = f32(base), f32(scale)
    log_base = f32(1) if base == -1 else f32(np.log(base))
    return float(f32(1) / log_base), float(scale / log_base)


def kernel_params(kind, q, backward=False):
    """(p0, p1, p2) of b2c_neuron_forward / _backward for the layer parameters q."""
    if kind == "ELU":
        return (q.get("alpha", 1.0), 0.0, 0.0)
    if kind == "POWER":
        return (q.get("power", 1.0), q.get("scale", 1.0), q.get("shift", 0.0))
    if kind == "EXP":
        inner, outer = exp_constants(q.get("base", -1.0), q.get("scale", 1.0), q.get("shift", 0.0))
        return (inner, outer, 0.0)
    if kind == "LOG":
        bs, bns = log_constants(q.get("base", -1.0), q.get("scale", 1.0))
        return (q.get("scale", 1.0), q.get("shift", 0.0), bns if backward else bs)
    if kind == "THRESHOLD":
        return (q.get("threshold", 0.0), 0.0, 0.0)
    return (0.0, 0.0, 0.0)


# ---- float64 closed forms -------------------------------------------------------------------------------------------------
def _base(q):
    b = q.get("base", -1.0)
    return np.e if b == -1 else b


def forward(kind, x, q):
    x = np.asarray(x, np.float64)
    if kind == "ELU":
        return np.where(x > 0, x, q.get("alpha", 1.0) * np.expm1(np.minimum(x, 0)))
    if kind == "POWER":
        p, a, b = q.get("power", 1.0), q.get("scale", 1.0), q.get("shift", 0.0)
        if p * a == 0:
            return np.full_like(x, 1.0 if p == 0 else b ** p)
        return np.power(b + a * x, p)
    if kind == "ABSVAL":
        return np.abs(x)
    if kind == "BNLL":
        return np.logaddexp(0.0, x)
    if kind == "EXP":
        return np.power(_base(q), q.get("shift", 0.0) + q.get("scale", 1.0) * x)
    if kind == "LOG":
        return np.log(q.get("shift", 0.0) + q.get("scale", 1.0) * x) / np.log(_base(q))
    if kind == "THRESHOLD":
        return (x > q.get("threshold", 0.0)).astype(np.float64)
    raise ValueError(kind)


def backward(kind, x, dy, q):
    """dx = dy * dy/dx at x (the derivative, not the reference's rewriting of it)."""
    x, dy = np.asarray(x, np.float64), np.asarray(dy, np.float64)
    if kind == "ELU":
        return dy * np.where(x > 0, 1.0, q.get("alpha", 1.0) * np.exp(np.minimum(x, 0)))
    if kind == "POWER":
        p, a, b = q.get("power", 1.0), q.get("scale", 1.0), q.get("shift", 0.0)
        if p * a == 0 or p == 1:
            return dy * (p * a)
        return dy * p * a * np.power(b + a * x, p - 1)
    if kind == "ABSVAL":
        return dy * np.sign(x)
    if kind == "BNLL":
        return dy / (1.0 + np.exp(-np.minimum(x, 50.0)))
    if kind == "EXP":
        return dy * np.log(_base(q)) * q.get("scale", 1.0) * forward(kind, x, q)
    if kind == "LOG":
        a = q.get("scale", 1.0)
        return dy * a / ((q.get("shift", 0.0) + a * x) * np.log(_base(q)))
    raise ValueError(kind)


def prelu_forward(x, slope, shared=False):
    x = np.asarray(x, np.float64)
    s = np.asarray(slope, np.float64).reshape(-1)
    s = np.full(x.shape[1], s[0]) if shared else s
    sb = s.reshape((1, -1) + (1,) * (x.ndim - 2))
    return np.where(x > 0, x, x * sb)


def prelu_backward(x, dy, slope, shared=False):
    """(dx, dslope, sum |dslope terms| per slope entry) in float64."""
    x, dy = np.asarray(x, np.float64), np.asarray(dy, np.float64)
    s = np.asarray(slope, np.float64).reshape(-1)
    s = np.full(x.shape[1], s[0]) if shared else s
    sb = s.reshape((1, -1) + (1,) * (x.ndim - 2))
    dx = dy * np.where(x > 0, 1.0, sb)
    terms = dy * x * (x <= 0)
    axes = tuple(a for a in range(x.ndim) if a != 1)
    ds, mag = terms.sum(axis=axes), np.abs(terms).sum(axis=axes)
    if shared:
        ds, mag = np.array([ds.sum()]), np.array([mag.sum()])
    return dx, ds, mag


# ---- float32 restatements of the rules the kernels compute exactly ------------------------------------------------------------
def forward_f32(kind, x, p):
    x = np.asarray(x, f32)
    p0, p1, p2 = (f32(v) for v in p)
    if kind == "ABSVAL":
        return np.abs(x)
    if kind == "THRESHOLD":
        return (x > p0).astype(f32)
    if kind == "POWER" and p0 in (1, 2):
        ds = f32(p0 * p1)
        if ds == 0:
            return np.full_like(x, f32(1) if p0 == 0 else f32(p2 ** p0))
        t = x.copy()
        if p1 != 1:
            t = (p1 * t).astype(f32)
        if p2 != 0:
            t = (t + p2).astype(f32)
        return t if p0 == 1 else (t * t).astype(f32)
    raise ValueError(kind)


def backward_f32(kind, x, y, dy, p):
    x, dy = np.asarray(x, f32), np.asarray(dy, f32)
    p0, p1, p2 = (f32(v) for v in p)
    if kind == "ABSVAL":
        return (np.sign(x).astype(f32) * dy).astype(f32)
    if kind == "POWER" and p0 in (1, 2):
        ds = f32(p0 * p1)
        if ds == 0 or p0 == 1:
            return (dy * ds).astype(f32)
        g = (f32(ds * p1) * x).astype(f32)
        if p2 != 0:
            g = (g + f32(ds * p2)).astype(f32)
        return (dy * g).astype(f32)
    raise ValueError(kind)


def prelu_forward_f32(x, slope, shared=False):
    x = np.asarray(x, f32)
    s = np.asarray(slope, f32).reshape(-1)
    s = np.full(x.shape[1], s[0], f32) if shared else s
    sb = s.reshape((1, -1) + (1,) * (x.ndim - 2))
    return np.where(x > 0, x, (x * sb).astype(f32)).astype(f32)


def prelu_dx_f32(x, dy, slope, shared=False):
    x, dy = np.asarray(x, f32), np.asarray(dy, f32)
    s = np.asarray(slope, f32).reshape(-1)
    s = np.full(x.shape[1], s[0], f32) if shared else s
    sb = s.reshape((1, -1) + (1,) * (x.ndim - 2))
    gain = ((x > 0).astype(f32) + ((x <= 0).astype(f32) * sb).astype(f32)).astype(f32)
    return (dy * gain).astype(f32)


# ---- the neuron net: conv -> in-place PReLU -> conv -> ELU -> Power -> AbsVal -> BNLL -> Exp -> Log -> InnerProduct -> loss ------
NET_Q = {"elu": {"alpha": 0.7}, "pow": {"power": 2.0, "scale": 0.5, "shift": 0.25}, "exp": {"base": 2.0, "scale": 0.25, "shift": -0.5},
         "log": {"base": 10.0, "scale": 0.5, "shift": 1.5}, "thr": {"threshold": 0.3}}


def net_prototxt(N, H, W, classes, shared, prelu_in_place=True):
    sh = " channel_shared: true" if shared else ""
    top = "c1" if prelu_in_place else "pr"
    return (
        'name: "neuron_net"\n'
        f'layer {{ name: "data" type: "Input" top: "data" top: "label" input_param {{ shape {{ dim: {N} dim: 3 dim: {H} dim: {W} }} '
        f'shape {{ dim: {N} }} }} }}\n'
        'layer { name: "c1" type: "Convolution" bottom: "data" top: "c1" convolution_param { num_output: 6 kernel_size: 3 pad: 1 } }\n'
        f'layer {{ name: "pr" type: "PReLU" bottom: "c1" top: "{top}" prelu_param {{ filler {{ type: "constant" value: 0.3 }}{sh} }} }}\n'
        f'layer {{ name: "c2" type: "Convolution" bottom: "{top}" top: "c2" convolution_param {{ num_output: 4 kernel_size: 3 pad: 1 }} }}\n'
        'layer { name: "elu" type: "ELU" bottom: "c2" top: "elu" elu_param { alpha: 0.7 } }\n'
        'layer { name: "pow" type: "Power" bottom: "elu" top: "pow" power_param { power: 2 scale: 0.5 shift: 0.25 } }\n'
        'layer { name: "abs" type: "AbsVal" bottom: "pow" top: "abs" }\n'
        'layer { name: "bnll" type: "BNLL" bottom: "abs" top: "bnll" }\n'
        'layer { name: "exp" type: "Exp" bottom: "bnll" top: "exp" exp_param { base: 2 scale: 0.25 shift: -0.5 } }\n'
        'layer { name: "log" type: "Log" bottom: "exp" top: "log" log_param { base: 10 scale: 0.5 shift: 1.5 } }\n'
        f'layer {{ name: "fc" type: "InnerProduct" bottom: "log" top: "fc" inner_product_param {{ num_output: {classes} }} }}\n'
        'layer { name: "loss" type: "SoftmaxWithLoss" bottom: "fc" bottom: "label" top: "loss" }\n'
        'layer { name: "thr" type: "Threshold" bottom: "c2" top: "thr" threshold_param { threshold: 0.3 } }\n')


def net_param_shapes(H, W, classes, shared):
    """learnable ids in layer order: c1 w, b; pr slope; c2 w, b; fc w, b"""
    return [(6, 3, 3, 3), (6,), () if shared else (6,), (4, 6, 3, 3), (4,), (classes, 4 * H * W), (classes,)]


def net_forward_backward(params, x, label):
    """float64: (loss, [gradients in learnable-id order], {blob name: value})"""
    import torch
    import torch.nn.functional as F
    P = [torch.tensor(np.asarray(p, np.float64), requires_grad=True) for p in params]
    X = torch.tensor(np.asarray(x, np.float64))
    c1 = F.conv2d(X, P[0], P[1], padding=1)
    s = P[2].reshape(-1)
    pr = torch.where(c1 > 0, c1, c1 * (s.reshape(1, -1, 1, 1) if s.numel() > 1 else s))
    c2 = F.conv2d(pr, P[3], P[4], padding=1)
    q = NET_Q
    elu = torch.where(c2 > 0, c2, q["elu"]["alpha"] * torch.expm1(torch.clamp(c2, max=0)))
    pw = (q["pow"]["shift"] + q["pow"]["scale"] * elu) ** q["pow"]["power"]
    ab = pw.abs()
    bn = F.softplus(ab)
    ex = q["exp"]["base"] ** (q["exp"]["shift"] + q["exp"]["scale"] * bn)
    lg = torch.log(q["log"]["shift"] + q["log"]["scale"] * ex) / np.log(q["log"]["base"])
    fc = lg.reshape(lg.shape[0], -1) @ P[5].T + P[6]
    lab = torch.tensor(np.asarray(label).astype(np.int64))
    loss = F.cross_entropy(fc, lab)
    loss.backward()
    blobs = {"c1": pr, "c2": c2, "elu": elu, "pow": pw, "abs": ab, "bnll": bn, "exp": ex, "log": lg, "fc": fc,
             "thr": (c2 > q["thr"]["threshold"]).double()}
    return float(loss), [p.grad.numpy().copy() for p in P], {k: v.detach().numpy() for k, v in blobs.items()}

"""Layer-by-layer float64 checker of one TrainNet forward_backward() on a whole prototxt net (tests/test_fullnet_parity_*.py).

Teacher forcing: every layer's tops are recomputed in float64 from the PRODUCT's own bottoms and parameters, every bottom diff
from the product's own top diffs, so errors do not compound over 50 layers and a near-tie in a max pool or a ReLU cannot flip a
decision between the two sides.  An in-place layer (ReLU, Dropout) belongs to the unit of the layer that produced its blob: the
blob the product keeps is the chain's output, and its diff is the chain's input gradient.

The net is read from its prototxt text (the product parses the same text).  The caller supplies the product's state:
  fetch(blob, diff) -> flat float32 array of a blob's data or diff after forward_backward()
  params[layer]     -> [(data, diff), ...] in the layer's blob order (conv w [, b]; BatchNorm scale, shift; InnerProduct w, b)
and gets back a list of Check records.  TEST INFRASTRUCTURE ONLY."""
import re
from dataclasses import dataclass

import numpy as np

from oracle import layers_oracle as lo

# Per-tensor bars, max|got - ref| / max|ref| (0: bit equality).  Conv / InnerProduct: the fp32-mode bar of the conv suites (the
# tensor-core kernels run 3xBF16 / 3xTF32 split products, ~1e-6 relative per dot product).  BatchNorm, AVE pooling, LRN and the
# softmax loss accumulate in fp32 (or better) over at most N*H*W terms per value, ~1e-6 relative; 1e-5 is their suites' bar.
# MAX pooling backward adds at most ceil(k/s)^2 selected fp32 values per bottom element, in an order of its own; the worst geometry
# run here is GoogLeNet's 3x3 / stride-1 inception pools, 9 terms: the difference to the float64 sum is at most
# 8 * 2^-24 * 9 max|dy| < 4.3e-6 max|dy|.  The bottom element that receives the largest |dy| holds it plus at most 8 others, and
# the bottoms of these pools are post-ReLU maps whose gradient is spread thinly, so max|ref| is of the order of max|dy|; the bar
# is 1e-5 of max|ref| (measured worst on the four nets: 1e-7).
# ReLU and Dropout run in place, so the product never keeps their input or their output gradient apart from the chain's: their
# exact checks are the masks (no negative value leaves a ReLU, a ReLU-cut or dropped position holds exactly 0 in data and diff);
# the values that survive a mask are checked at the bar of the layer that produced the blob.
BAR = {"Convolution": 1e-4, "InnerProduct": 1e-4, "BatchNorm": 1e-5, "AVE": 1e-5, "MAX": 1e-5, "LRN": 1e-5,
       "SoftmaxWithLoss": 1e-5, "Eltwise": 0.0, "Concat": 0.0}
LOSS_BAR = 1e-6                 # each loss top against float64 softmax-loss of the product's logits, relative
IN_PLACE = ("ReLU", "Dropout")


@dataclass
class Check:
    layer: str
    kind: str        # layer kind of the bar: Convolution, BatchNorm, MAX, AVE, ..., or ReLU / Dropout for the exact mask checks
    what: str        # "y" (forward top), "dx:<blob>", "dW", "db", "dgamma", "dbeta", "loss", "mask_fwd", "mask_bwd"
    err: float       # relative error (exact checks: number of mismatching elements)
    bar: float

    @property
    def ok(self):
        return np.isfinite(self.err) and self.err <= self.bar


# ------------------------------------------------------------------------------------------------------------ prototxt
def _tokens(text):
    text = re.sub(r"#[^\n]*", "", text)
    return re.findall(r'"[^"]*"|[{}:]|[^\s{}:"]+', text)


def _parse_block(toks, i):
    out = []
    while i < len(toks) and toks[i] != "}":
        key = toks[i]
        i += 1
        if toks[i] == ":":
            i += 1
        if toks[i] == "{":
            val, i = _parse_block(toks, i + 1)
            i += 1
        else:
            val = toks[i].strip('"')
            i += 1
        out.append((key, val))
    return out, i


def _get(block, key, default=None, cast=None):
    for k, v in block:
        if k == key:
            return cast(v) if cast else v
    return default


def _all(block, key):
    return [v for k, v in block if k == key]


def parse_layers(prototxt):
    """[dict(name, type, bottom, top, ...)] of a TRAIN-phase net, in prototxt order, with the fields this checker reads."""
    top, _ = _parse_block(_tokens(prototxt), 0)
    layers = []
    for blk in _all(top, "layer"):
        L = dict(name=_get(blk, "name"), type=_get(blk, "type"), bottom=_all(blk, "bottom"), top=_all(blk, "top"),
                 loss_weight=_get(blk, "loss_weight", None, float))
        t = L["type"]
        if t == "Convolution":
            cp = _get(blk, "convolution_param")
            L.update(o=_get(cp, "num_output", cast=int), k=_get(cp, "kernel_size", cast=int), s=_get(cp, "stride", 1, int),
                     p=_get(cp, "pad", 0, int), g=_get(cp, "group", 1, int), bias=_get(cp, "bias_term", "true") == "true")
        elif t == "Pooling":
            pp = _get(blk, "pooling_param")
            L.update(m=_get(pp, "pool", "MAX"), k=_get(pp, "kernel_size", cast=int), s=_get(pp, "stride", 1, int),
                     p=_get(pp, "pad", 0, int))
        elif t == "LRN":
            lp = _get(blk, "lrn_param", [])
            L.update(size=_get(lp, "local_size", 5, int), alpha=_get(lp, "alpha", 1.0, float), beta=_get(lp, "beta", 0.75, float),
                     k=_get(lp, "k", 1.0, float))
        elif t == "Dropout":
            L.update(ratio=_get(_get(blk, "dropout_param", []), "dropout_ratio", 0.5, float))
        elif t == "BatchNorm":
            L.update(eps=_get(_get(blk, "batch_norm_param", []), "eps", 1e-5, float))
        elif t == "Eltwise":
            assert _get(_get(blk, "eltwise_param", []), "operation", "SUM") == "SUM", "only Eltwise SUM is checked"
        elif t == "SoftmaxWithLoss" and L["loss_weight"] is None:
            L["loss_weight"] = 1.0
        layers.append(L)
    return layers


def units(layers):
    """[(producer index, [in-place layer indices on its first top])], in execution order; Input layers are skipped."""
    out = []
    for i, L in enumerate(layers):
        if L["type"] in ("Input",) or (L["type"] in IN_PLACE and L["bottom"] == L["top"]):
            continue
        chain = [j for j in range(i + 1, len(layers)) if layers[j]["type"] in IN_PLACE and layers[j]["bottom"] == [L["top"][0]]
                 and layers[j]["top"] == [L["top"][0]]]
        out.append((i, chain))
    return out


def dropout_stream(seed, layer_index):
    """TrainNet's dropout seed of layer `layer_index` of a trainer seeded `seed` (netoracle's formula)"""
    return (int(seed) * 0x100000001B3 + layer_index) & 0xFFFFFFFFFFFFFFFF


# ------------------------------------------------------------------------------------------------------------ float64 layers
def _torch():
    import torch
    return torch


def conv_forward(x, w, b, s, p, g):
    torch = _torch()
    y = torch.nn.functional.conv2d(torch.from_numpy(np.asarray(x, np.float64)), torch.from_numpy(np.asarray(w, np.float64)),
                                   None if b is None else torch.from_numpy(np.asarray(b, np.float64)), stride=s, padding=p, groups=g)
    return y.numpy()


def conv_backward(x, w, dy, s, p, g, want_dx=True):
    """-> (dW, db, dx or None), float64"""
    torch = _torch()
    X = torch.from_numpy(np.asarray(x, np.float64)).requires_grad_(want_dx)
    W = torch.from_numpy(np.asarray(w, np.float64)).requires_grad_(True)
    DY = torch.from_numpy(np.asarray(dy, np.float64))
    torch.nn.functional.conv2d(X, W, None, stride=s, padding=p, groups=g).backward(DY)
    return W.grad.numpy(), DY.sum(dim=(0, 2, 3)).numpy(), X.grad.numpy() if want_dx else None


def bn_forward(x, gamma, beta, eps):
    x = x.astype(np.float64)
    mean = x.mean(axis=(0, 2, 3), keepdims=True)
    var = ((x - mean) ** 2).mean(axis=(0, 2, 3), keepdims=True)
    xn = (x - mean) / np.sqrt(var + eps)
    return xn * gamma.reshape(1, -1, 1, 1) + beta.reshape(1, -1, 1, 1), xn, 1.0 / np.sqrt(var + eps)


def bn_backward(dy, xn, gamma, invstd):
    dy = dy.astype(np.float64)
    m = dy.size / dy.shape[1]
    dg = (dy * xn).sum(axis=(0, 2, 3))
    db = dy.sum(axis=(0, 2, 3))
    dx = gamma.reshape(1, -1, 1, 1) * invstd * (dy - (db / m).reshape(1, -1, 1, 1) - xn * (dg / m).reshape(1, -1, 1, 1))
    return dg, db, dx


def _pool_geometry(H, W, k, s, p):
    Ho, Wo = lo.pooled_extent(H, k, s, p), lo.pooled_extent(W, k, s, p)
    ph_hi = max(0, (Ho - 1) * s + k - H - p)
    pw_hi = max(0, (Wo - 1) * s + k - W - p)
    return Ho, Wo, ph_hi, pw_hi


def max_pool_forward(x, k, s, p):
    """-> (y in x's dtype, flat argmax index into H*W): the first maximum of each window in row-major order (a strict '>' scan)"""
    N, C, H, W = x.shape
    Ho, Wo, ph, pw = _pool_geometry(H, W, k, s, p)
    xp = np.full((N, C, H + p + ph, W + p + pw), -np.inf, x.dtype)
    xp[:, :, p:p + H, p:p + W] = x
    best = np.full((N, C, Ho, Wo), -np.inf, x.dtype)
    arg = np.zeros((N, C, Ho, Wo), np.int64)
    hh = np.arange(Ho)[:, None] * s - p
    ww = np.arange(Wo)[None, :] * s - p
    for i in range(k):
        for j in range(k):
            v = xp[:, :, i:i + s * (Ho - 1) + 1:s, j:j + s * (Wo - 1) + 1:s]
            take = v > best
            best = np.where(take, v, best)
            arg = np.where(take, (hh + i) * W + (ww + j), arg)
    return best, arg


def max_pool_backward(dy, arg, x_shape):
    N, C, H, W = x_shape
    dx = np.zeros((N * C, H * W), np.float64)
    rows = np.repeat(np.arange(N * C), dy.shape[2] * dy.shape[3])
    np.add.at(dx, (rows, arg.reshape(-1)), dy.astype(np.float64).reshape(-1))
    return dx.reshape(x_shape)


def _ave_divisor(H, W, Ho, Wo, k, s, p):
    hs = np.arange(Ho) * s - p
    ws = np.arange(Wo) * s - p
    dh = np.minimum(hs + k, H + p) - hs
    dw = np.minimum(ws + k, W + p) - ws
    return (dh[:, None] * dw[None, :]).astype(np.float64)


def ave_pool_forward(x, k, s, p):
    N, C, H, W = x.shape
    Ho, Wo, ph, pw = _pool_geometry(H, W, k, s, p)
    xp = np.zeros((N, C, H + p + ph, W + p + pw), np.float64)
    xp[:, :, p:p + H, p:p + W] = x
    acc = np.zeros((N, C, Ho, Wo), np.float64)
    for i in range(k):
        for j in range(k):
            acc += xp[:, :, i:i + s * (Ho - 1) + 1:s, j:j + s * (Wo - 1) + 1:s]
    return acc / _ave_divisor(H, W, Ho, Wo, k, s, p)


def ave_pool_backward(dy, x_shape, k, s, p):
    N, C, H, W = x_shape
    Ho, Wo, ph, pw = _pool_geometry(H, W, k, s, p)
    g = dy.astype(np.float64) / _ave_divisor(H, W, Ho, Wo, k, s, p)
    dxp = np.zeros((N, C, H + p + ph, W + p + pw), np.float64)
    for i in range(k):
        for j in range(k):
            dxp[:, :, i:i + s * (Ho - 1) + 1:s, j:j + s * (Wo - 1) + 1:s] += g
    return dxp[:, :, p:p + H, p:p + W]


def lrn_forward(x, size, alpha, beta, k):
    x = x.astype(np.float64)
    C = x.shape[1]
    sq = np.concatenate([np.zeros((x.shape[0], 1) + x.shape[2:]), np.cumsum(x * x, axis=1)], axis=1)
    lo_ = np.clip(np.arange(C) - (size - 1) // 2, 0, C)
    hi_ = np.clip(np.arange(C) - (size - 1) // 2 + size, 0, C)
    scale = k + (sq[:, hi_] - sq[:, lo_]) * alpha / size
    return x * scale ** (-beta), scale


def lrn_backward(x, y, scale, dy, size, alpha, beta):
    x, dy = x.astype(np.float64), dy.astype(np.float64)
    C = x.shape[1]
    ratio = dy * y / scale
    cs = np.concatenate([np.zeros((x.shape[0], 1) + x.shape[2:]), np.cumsum(ratio, axis=1)], axis=1)
    ipp = size - (size + 1) // 2
    lo_ = np.clip(np.arange(C) - ipp, 0, C)
    hi_ = np.clip(np.arange(C) - ipp + size, 0, C)
    return dy * scale ** (-beta) - 2.0 * alpha * beta / size * x * (cs[:, hi_] - cs[:, lo_])


def softmax_loss(logits, labels, loss_weight):
    """-> (loss, d logits), float64, VALID normalisation over the batch"""
    z = logits.astype(np.float64).reshape(len(labels), -1)
    z = z - z.max(axis=1, keepdims=True)
    prob = np.exp(z)
    prob /= prob.sum(axis=1, keepdims=True)
    lab = labels.astype(np.int64)
    loss = -np.log(prob[np.arange(len(lab)), lab]).mean()
    d = prob.copy()
    d[np.arange(len(lab)), lab] -= 1.0
    return loss, d * (loss_weight / len(lab))


# ------------------------------------------------------------------------------------------------------------ the walk
def rel(got, ref):
    got = np.asarray(got, np.float64).reshape(-1)
    ref = np.asarray(ref, np.float64).reshape(-1)
    if got.size != ref.size or not np.isfinite(got).all():
        return float("inf")
    den = float(np.max(np.abs(ref))) if ref.size else 0.0
    num = float(np.max(np.abs(got - ref))) if ref.size else 0.0
    return num / den if den > 0 else (0.0 if num == 0 else float("inf"))


def mismatches(got, ref):
    got = np.asarray(got, np.float32).reshape(-1)
    ref = np.asarray(ref, np.float32).reshape(-1)
    if got.size != ref.size:
        return float("inf")
    return float(np.count_nonzero((got != ref) | np.isnan(got)))       # value equality: a masked -0.0 equals 0.0


def _kind(L):
    return L["m"] if L["type"] == "Pooling" else L["type"]


def walk(layers, fetch, params, input_shape, labels, seed=1701, iteration=0, forward_only=False, kinds=None, shapes=None):
    """Check one forward_backward() of the net `layers` (parse_layers) whose product state `fetch` / `params` expose.
    forward_only: forward tops only; kinds: restrict the checks to these layer types.  shapes: a dict the blob shapes are stored in;
    when it already holds them (an earlier walk of the same net), units outside `kinds` are not recomputed.  Returns [Check]."""
    checks = []
    known = dict(shapes) if shapes else {}
    shape = {layers[0]["top"][0]: tuple(input_shape)} if layers[0]["type"] == "Input" else {}
    cache = {}

    def data(name):
        if ("d", name) not in cache:
            cache[("d", name)] = fetch(name, False).reshape(shape[name])
        return cache[("d", name)]

    def diff(name):
        if ("g", name) not in cache:
            cache[("g", name)] = fetch(name, True).reshape(shape[name])
        return cache[("g", name)]

    def want(L):
        return kinds is None or L["type"] in kinds

    ulist = units(layers)
    masks = {}                         # dropout layer index -> float32 mask
    bottom_contrib = {}                # blob -> [(float64 contribution, bar, exact float32 contribution or None)]
    # ---------------------------------------------------------------------------------------------------- forward
    for i, chain in ulist:
        L = layers[i]
        t, kind = L["type"], _kind(L)
        if not want(L) and L["top"][0] in known:
            shape[L["top"][0]] = known[L["top"][0]]
            continue
        xs = [data(b) for b in L["bottom"] if b in shape]
        exact = None                   # float32 top the product must equal bit for bit
        if t == "Convolution":
            w, b = [p[0] for p in params[L["name"]]] + [None] * (2 - len(params[L["name"]]))
            w = w.reshape(L["o"], xs[0].shape[1] // L["g"], L["k"], L["k"])
            ref = conv_forward(xs[0], w, b, L["s"], L["p"], L["g"])
        elif t == "BatchNorm":
            g_, b_ = (p[0] for p in params[L["name"]])
            ref, _, _ = bn_forward(xs[0], g_, b_, L["eps"])
        elif t == "InnerProduct":
            w, b = (p[0] for p in params[L["name"]])
            x2 = xs[0].reshape(xs[0].shape[0], -1).astype(np.float64)
            ref = x2 @ w.reshape(-1, x2.shape[1]).astype(np.float64).T + b.astype(np.float64)
        elif t == "Pooling" and L["m"] == "MAX":
            exact, _ = max_pool_forward(xs[0], L["k"], L["s"], L["p"])
            ref = exact.astype(np.float64)
        elif t == "Pooling":
            ref = ave_pool_forward(xs[0], L["k"], L["s"], L["p"])
        elif t == "LRN":
            ref, _ = lrn_forward(xs[0], L["size"], L["alpha"], L["beta"], L["k"])
        elif t == "Eltwise":
            exact = xs[0].astype(np.float32)
            for x in xs[1:]:
                exact = exact + x.astype(np.float32)
            ref = exact.astype(np.float64)
        elif t == "Concat":
            exact = np.concatenate([x.astype(np.float32) for x in xs], axis=1)
            ref = exact.astype(np.float64)
        elif t == "SoftmaxWithLoss":
            loss, _ = softmax_loss(xs[0], labels, L["loss_weight"])
            shape[L["top"][0]] = (1,)
            if want(L):
                got = float(data(L["top"][0])[0])
                checks.append(Check(L["name"], t, "loss", abs(got - loss) / abs(loss) if np.isfinite(got) else float("inf"), LOSS_BAR))
            continue
        else:
            raise AssertionError(f"layer type {t} ({L['name']}) is not covered by the checker")
        top = L["top"][0]
        shape[top] = ref.shape
        for j in chain:                                  # the in-place chain, in order
            C_ = layers[j]
            if C_["type"] == "ReLU":
                ref = np.maximum(ref, 0.0)
                if exact is not None:
                    exact = np.maximum(exact, np.float32(0))
            else:
                m = lo.dropout_mask(int(np.prod(ref.shape)), C_["ratio"], dropout_stream(seed, j),
                                    iteration * int(np.prod(ref.shape))).reshape(ref.shape)
                masks[j] = m
                ref = ref * m
                if exact is not None:
                    exact = exact * m
        if not want(L):
            continue
        got = data(top)
        if exact is not None and BAR[kind] == 0.0:
            checks.append(Check(L["name"], kind, "y", mismatches(got, exact), 0.0))
        elif exact is not None and kind == "MAX":        # a selection: bit equality
            checks.append(Check(L["name"], kind, "y", mismatches(got, exact), 0.0))
        else:
            checks.append(Check(L["name"], kind, "y", rel(got, ref), BAR[kind]))
        for j in chain:                                  # the masks are exact: no negative value escapes a ReLU, dropout zeros stay
            if layers[j]["type"] == "ReLU":
                checks.append(Check(layers[j]["name"], "ReLU", "mask_fwd", float(np.count_nonzero(got < 0)), 0.0))
            else:
                checks.append(Check(layers[j]["name"], "Dropout", "mask_fwd", float(np.count_nonzero(got[masks[j] == 0] != 0)), 0.0))
    if shapes is not None:
        shapes.update(shape)
    if forward_only:
        return checks
    # ---------------------------------------------------------------------------------------------------- backward
    def add(blob, contrib, bar, exact=None):
        bottom_contrib.setdefault(blob, []).append((contrib, bar, exact))

    for i, chain in reversed(ulist):
        L = layers[i]
        t, kind = L["type"], _kind(L)
        top = L["top"][0]
        bots = [b for b in L["bottom"] if b in shape and not (t == "SoftmaxWithLoss" and b != L["bottom"][0])]
        needs_dx = [b != layers[0]["top"][0] for b in bots]     # the net input takes no gradient
        if t == "SoftmaxWithLoss":
            _, d = softmax_loss(data(bots[0]), labels, L["loss_weight"])
            add(bots[0], d.reshape(shape[bots[0]]), BAR[t])
            continue
        dy = diff(top)
        if t == "Convolution":
            prm = params[L["name"]]
            x = data(bots[0])
            w = prm[0][0].reshape(L["o"], x.shape[1] // L["g"], L["k"], L["k"])
            dw, db, dx = conv_backward(x, w, dy, L["s"], L["p"], L["g"], needs_dx[0])
            if want(L):
                checks.append(Check(L["name"], t, "dW", rel(prm[0][1], dw), BAR[t]))
                if len(prm) > 1:
                    checks.append(Check(L["name"], t, "db", rel(prm[1][1], db), BAR[t]))
            if needs_dx[0]:
                add(bots[0], dx, BAR[t])
        elif t == "BatchNorm":
            (g_, dg_got), (b_, db_got) = params[L["name"]]
            _, xn, invstd = bn_forward(data(bots[0]), g_, b_, L["eps"])
            dg, dbt, dx = bn_backward(dy, xn, g_.astype(np.float64), invstd)
            if want(L):
                checks.append(Check(L["name"], t, "dgamma", rel(dg_got, dg), BAR[t]))
                checks.append(Check(L["name"], t, "dbeta", rel(db_got, dbt), BAR[t]))
            add(bots[0], dx, BAR[t])
        elif t == "InnerProduct":
            (w, dw_got), (b, db_got) = params[L["name"]]
            x = data(bots[0])
            x2 = x.reshape(x.shape[0], -1).astype(np.float64)
            d64 = dy.reshape(x.shape[0], -1).astype(np.float64)
            if want(L):
                checks.append(Check(L["name"], t, "dW", rel(dw_got, d64.T @ x2), BAR[t]))
                checks.append(Check(L["name"], t, "db", rel(db_got, d64.sum(axis=0)), BAR[t]))
            if needs_dx[0]:
                add(bots[0], (d64 @ w.reshape(d64.shape[1], -1).astype(np.float64)).reshape(x.shape), BAR[t])
        elif t == "Pooling" and L["m"] == "MAX":
            x = data(bots[0])
            _, arg = max_pool_forward(x, L["k"], L["s"], L["p"])
            add(bots[0], max_pool_backward(dy, arg, x.shape), BAR["MAX"])
        elif t == "Pooling":
            add(bots[0], ave_pool_backward(dy, shape[bots[0]], L["k"], L["s"], L["p"]), BAR["AVE"])
        elif t == "LRN":
            x = data(bots[0])
            y, scale = lrn_forward(x, L["size"], L["alpha"], L["beta"], L["k"])
            add(bots[0], lrn_backward(x, y, scale, dy, L["size"], L["alpha"], L["beta"]), BAR[t])
        elif t == "Eltwise":
            for b in bots:
                add(b, dy.astype(np.float64), 0.0, dy)
        elif t == "Concat":
            c0 = 0
            for b in bots:
                cb = shape[b][1]
                add(b, dy[:, c0:c0 + cb].astype(np.float64), 0.0, dy[:, c0:c0 + cb])
                c0 += cb
    # every blob's diff: the sum over its consumers, then the backward of its in-place chain (Dropout, then ReLU)
    chain_of = {layers[i]["top"][0]: (i, chain) for i, chain in ulist}
    for blob, parts in bottom_contrib.items():
        i, chain = chain_of[blob]
        L = layers[i]
        if not want(L):
            continue
        ref = sum(p[0] for p in parts)
        bar = max(p[1] for p in parts)
        exact = parts[0][2] if len(parts) == 1 and parts[0][2] is not None else None
        got_data = data(blob)
        for j in reversed(chain):
            if layers[j]["type"] == "Dropout":
                ref = ref * masks[j]
                exact = None if exact is None else exact * masks[j]
            else:                                        # the mask of an in-place ReLU is (its blob's final data > 0)
                ref = np.where(got_data > 0, ref, 0.0)
                exact = None if exact is None else np.where(got_data > 0, exact, np.float32(0))
        got = diff(blob)
        kinds_ = "+".join(sorted({k for k in (_kind(layers[c]) for c in consumers(layers, blob))}))
        if exact is not None:
            checks.append(Check(L["name"], kinds_, "dx:" + blob, mismatches(got, exact), 0.0))
        else:
            checks.append(Check(L["name"], kinds_, "dx:" + blob, rel(got, ref), bar))
        for j in chain:
            if layers[j]["type"] == "ReLU":
                checks.append(Check(layers[j]["name"], "ReLU", "mask_bwd", float(np.count_nonzero(got[got_data <= 0] != 0)), 0.0))
            else:
                checks.append(Check(layers[j]["name"], "Dropout", "mask_bwd", float(np.count_nonzero(got[masks[j] == 0] != 0)), 0.0))
    return checks


def consumers(layers, blob):
    return [i for i, L in enumerate(layers) if blob in L["bottom"] and not (L["type"] in IN_PLACE and L["top"] == L["bottom"])]


def summary(checks):
    """{(kind, what class, bar): worst error} -- the per-kind report of a run"""
    out = {}
    for c in checks:
        w = "dx" if c.what.startswith("dx:") else c.what
        key = (c.kind, w, c.bar)
        out[key] = max(out.get(key, 0.0), c.err)
    return out


def failures(checks):
    return [c for c in checks if not c.ok]

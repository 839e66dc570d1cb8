"""float64 statements of SoftmaxWithLoss and Accuracy over an [outer, C, inner] view (softmax_loss_layer.cpp:44-160,
accuracy_layer.cpp:21-101): one softmax over C per (outer, inner) pixel, loss_param's ignore_label and normalization, and the
per-class accuracy.  Labels are float class ids read as int."""
import numpy as np

NORMS = ("FULL", "VALID", "BATCH_SIZE", "NONE")


def view(shape, axis):
    axis = axis % len(shape)
    outer = int(np.prod(shape[:axis], dtype=np.int64))
    inner = int(np.prod(shape[axis + 1:], dtype=np.int64))
    return outer, shape[axis], inner


def softmax(x, axis=1):
    z = x.astype(np.float64)
    z = z - z.max(axis=axis, keepdims=True)
    e = np.exp(z)
    return e / e.sum(axis=axis, keepdims=True)


def normalizer(mode, outer, inner, valid, has_ignore):
    """get_normalizer (softmax_loss_layer.cpp:65-92), floored at 1."""
    n = {"FULL": outer * inner, "VALID": valid if has_ignore else outer * inner, "BATCH_SIZE": outer, "NONE": 1}[mode]
    return max(1.0, float(n))


def _pixels(x, labels, axis):
    outer, C, inner = view(x.shape, axis)
    return outer, C, inner, labels.reshape(outer, inner).astype(np.float64).astype(np.int64)


def softmax_loss(x, labels, axis=1, ignore_label=None, norm="VALID", loss_weight=1.0):
    """(loss, normalizer, prob [outer, C, inner], dx shaped like x) in float64.  An out-of-range label that is not ignored reads
    the nearest class in the loss and subtracts nothing in dx (the kernels' documented behaviour)."""
    outer, C, inner, lab = _pixels(x, labels, axis)
    p = softmax(x.reshape(outer, C, inner), axis=1)
    keep = np.ones_like(lab, bool) if ignore_label is None else lab != ignore_label
    cl = np.clip(lab, 0, C - 1)
    pl = np.take_along_axis(p, cl[:, None, :], axis=1)[:, 0, :]
    terms = -np.log(np.maximum(pl, np.finfo(np.float32).tiny))
    valid = int(keep.sum())
    nrm = normalizer(norm, outer, inner, valid, ignore_label is not None)
    loss = terms[keep].sum() / nrm
    onehot = (np.arange(C)[None, :, None] == lab[:, None, :]).astype(np.float64)
    dx = (p - onehot) * (loss_weight / nrm) * keep[:, None, :]
    return loss, nrm, p, dx.reshape(x.shape)


def loss_only(x, labels, **kw):
    return softmax_loss(x, labels, **kw)[0]


def accuracy(scores, labels, axis=1, top_k=1, ignore_label=None):
    """(accuracy, per_class[C]) as accuracy_layer.cpp: std::greater over (score, index) pairs, so on equal scores the larger index
    ranks first; ignored pixels skipped; accuracy / count (NaN for 0 / 0); per class hits / num or 0."""
    outer, C, inner, lab = _pixels(scores, labels, axis)
    z = scores.reshape(outer, C, inner).astype(np.float32)
    hits, count = 0, 0
    hc, nc = np.zeros(C), np.zeros(C)
    for o in range(outer):
        for i in range(inner):
            l = int(lab[o, i])
            if ignore_label is not None and l == ignore_label:
                continue
            count += 1
            if not 0 <= l < C:
                continue
            nc[l] += 1
            order = sorted(((float(z[o, k, i]), k) for k in range(C)), reverse=True)
            if l in [k for _, k in order[:top_k]]:
                hits += 1
                hc[l] += 1
    with np.errstate(invalid="ignore", divide="ignore"):
        acc = np.float32(hits) / np.float32(count) if count else np.float32(np.nan)
        per = np.where(nc == 0, 0.0, hc / np.where(nc == 0, 1, nc)).astype(np.float32)
    return np.float32(acc), per


def numeric_grad(f, x, eps=1e-2):
    """Central differences of a float64 scalar function over every element of x (GradientChecker's stepsize 1e-2)."""
    g = np.zeros_like(x, dtype=np.float64)
    xf = x.astype(np.float64).copy()
    flat = xf.reshape(-1)
    for k in range(flat.size):
        v = flat[k]
        flat[k] = v + eps
        up = f(xf)
        flat[k] = v - eps
        dn = f(xf)
        flat[k] = v
        g.reshape(-1)[k] = (up - dn) / (2 * eps)
    return g


# ---- a small FCN (the deconv_oracle encoder-decoder's pieces with a segmentation head) -----------------------------------------
#   data [N, 3, H, W] -> conv1 (4, 3x3 pad 1) -> pool (MAX 2x2 / 2) -> score (C, 1x1) -> up = Deconvolution (C, 4x4 / 2, group C,
#   bilinear, no bias, lr_mult 0: a frozen upsampler) -> [N, C, H + 2, W + 2] -> crop (Crop to data, axis 2, offset 1) -> [N, C, H, W]
#   -> SoftmaxWithLoss (ignore_label 255; the prob top) and Accuracy (ignore_label 255; the per-class top) against label [N, 1, H, W].
# Learnable blobs in layer order: conv1 w, b; score w, b; up w.
def fcn_layers(C=5, norm=""):
    """The layers after the data layer(s), bottoms `data` and `label`."""
    return f'''layer {{ name: "conv1" type: "Convolution" bottom: "data" top: "c1" convolution_param {{ num_output: 4 kernel_size: 3 pad: 1
  weight_filler {{ type: "gaussian" std: 0.01 }} }} }}
layer {{ name: "pool" type: "Pooling" bottom: "c1" top: "p1" pooling_param {{ pool: MAX kernel_size: 2 stride: 2 }} }}
layer {{ name: "score" type: "Convolution" bottom: "p1" top: "sc" convolution_param {{ num_output: {C} kernel_size: 1
  weight_filler {{ type: "gaussian" std: 0.1 }} }} }}
layer {{ name: "up" type: "Deconvolution" bottom: "sc" top: "up" param {{ lr_mult: 0 decay_mult: 0 }}
  convolution_param {{ num_output: {C} kernel_size: 4 stride: 2 group: {C} bias_term: false weight_filler {{ type: "bilinear" }} }} }}
layer {{ name: "crop" type: "Crop" bottom: "up" bottom: "data" top: "crop" crop_param {{ axis: 2 offset: 1 }} }}
layer {{ name: "loss" type: "SoftmaxWithLoss" bottom: "crop" bottom: "label" top: "loss" TOPS loss_param {{ ignore_label: 255 {norm} }} }}
layer {{ name: "acc" type: "Accuracy" bottom: "crop" bottom: "label" top: "acc" top: "per_class" accuracy_param {{ ignore_label: 255 }} }}
'''


def fcn_prototxt(N, H, W, C=5, norm="", prob_top=True):
    return (f'name: "fcn"\nlayer {{ name: "in" type: "Input" top: "data" top: "label" input_param {{ shape {{ dim: {N} dim: 3 dim: {H} dim: {W} }} '
            f'shape {{ dim: {N} dim: 1 dim: {H} dim: {W} }} }} }}\n' + fcn_layers(C, norm).replace("TOPS", 'top: "prob"' if prob_top else ""))


def fcn_param_shapes(C=5):
    return [(4, 3, 3, 3), (4,), (C, 4, 1, 1), (C,), (C, 1, 4, 4)]


def fcn_forward_backward(params, data, label, norm="VALID", loss_weight=1.0):
    """(loss, [gradient of each learnable blob], blobs) of fcn_prototxt in float64; params in the net's learnable order."""
    import deconv_oracle as do
    w1, b1, ws, bs, wu = [np.asarray(a, np.float64) for a in params]
    N, _, H, W = data.shape
    C = ws.shape[0]
    c1 = do._conv(data, w1, b1, 1, 1)
    win = c1.reshape(N, 4, H // 2, 2, W // 2, 2).transpose(0, 1, 2, 4, 3, 5).reshape(N, 4, H // 2, W // 2, 4)
    p1 = win.max(axis=-1)
    arg = win.argmax(axis=-1)                                     # the first maximum in (row, column) order, as the MAX kernel
    sc = do._conv(p1, ws, bs, 1, 0)
    up = do.deconv_forward(sc, wu, None, 4, 2, 0, 1, G=C)
    crop = up[:, :, 1:H + 1, 1:W + 1]
    loss, _, prob, dcrop = softmax_loss(crop, label, ignore_label=255, norm=norm, loss_weight=loss_weight)
    dup = np.zeros_like(up)
    dup[:, :, 1:H + 1, 1:W + 1] = dcrop
    dsc, dwu, _ = do.deconv_backward(sc, wu, dup, 4, 2, 0, 1, G=C)
    dp1, dws, dbs = do._conv_back(p1, ws, dsc, 1, 0)
    dwin = np.zeros(win.shape)
    np.put_along_axis(dwin, arg[..., None], dp1[..., None], axis=-1)
    dc1 = dwin.reshape(N, 4, H // 2, W // 2, 2, 2).transpose(0, 1, 2, 4, 3, 5).reshape(N, 4, H, W)
    _, dw1, db1 = do._conv_back(data, w1, dc1, 1, 1)
    return loss_weight * loss, [dw1, db1, dws, dbs, dwu], dict(c1=c1, p1=p1, sc=sc, up=up, crop=crop, prob=prob.reshape(crop.shape))

"""CPU oracle for the non-convolution layers on ResNet-50's path -- TEST INFRASTRUCTURE ONLY (numpy restatements of
the reference's *_cpu code; paths relative to /root/reference).  Parity status: pooling is PINNED by the reference's own known-answer vectors
(test_pooling_layer.cpp: TestForwardSquare / RectHigh / RectWide values and argmax masks, TestForwardMaxPadded,
TestForwardAve, the three TestSetup shapes), BatchNorm by the reference test's statistic (zero mean / unit variance per
channel), ReLU / InnerProduct / SoftmaxWithLoss by closed forms; every backward by finite differences, which is what
the reference's own GradientChecker tests do (it stores no golden gradients).  All in tests/test_layers_cpu.py."""
import numpy as np


# ReLULayer::Forward_cpu / Backward_cpu, src/caffe/layers/relu_layer.cpp:10-41
def relu_forward(x, slope=0.0):
    return np.maximum(x, 0) + slope * np.minimum(x, 0)


def relu_backward(dy, x, slope=0.0):
    return dy * ((x > 0) + slope * (x <= 0))


# BatchNormLayer::Forward_cpu (TRAIN), src/caffe/layers/batch_norm_layer.cpp:140-232
def bn_forward_train(x, gamma, beta, eps, maf, run_mean, run_var, first):
    x = x.astype(np.float32)
    ax = (0,) + tuple(range(2, x.ndim))
    shp = (1, -1) + (1,) * (x.ndim - 2)
    mean = x.mean(axis=ax, dtype=np.float64).astype(np.float32)
    xc = x - mean.reshape(shp)
    var_eps = (xc.astype(np.float64) ** 2).mean(axis=ax).astype(np.float32) + np.float32(eps)   # eps added before the average (:183-186)
    invstd = (1.0 / np.sqrt(var_eps)).astype(np.float32)
    xnorm = xc * invstd.reshape(shp)
    if first:                                    # iter_ <= 1: copy (:199-204)
        nm, nv = mean.copy(), var_eps.copy()
    else:
        nm = (1 - maf) * mean + maf * run_mean
        nv = (1 - maf) * var_eps + maf * run_var
    y = xnorm * gamma.reshape(shp) + beta.reshape(shp) if gamma is not None else xnorm.copy()
    return y.astype(np.float32), xnorm.astype(np.float32), mean, invstd, nm.astype(np.float32), nv.astype(np.float32)


# BatchNormLayer::Backward_cpu, batch_norm_layer.cpp:234-283 (scale/shift diffs are OVERWRITTEN, not accumulated)
def bn_backward(dy, xnorm, gamma, invstd):
    ax = (0,) + tuple(range(2, dy.ndim))
    shp = (1, -1) + (1,) * (dy.ndim - 2)
    dgamma = (dy.astype(np.float64) * xnorm).sum(axis=ax)
    dbeta = dy.astype(np.float64).sum(axis=ax)
    g = gamma.reshape(shp) if gamma is not None else 1.0
    cnt = dy.size / dy.shape[1]
    dx = g * invstd.reshape(shp) * (dy - (dbeta / cnt).reshape(shp) - xnorm * (dgamma / cnt).reshape(shp))
    return dgamma.astype(np.float32), dbeta.astype(np.float32), dx.astype(np.float32)


def pooled_extent(n, k, s, p):                   # PoolingLayer::Reshape: ceil mode with the last-window clip
    o = int(np.ceil((n + 2 * p - k) / s)) + 1
    if p > 0 and (o - 1) * s >= n + p:
        o -= 1
    return o


# PoolingLayer::Forward_cpu / Backward_cpu, src/caffe/layers/pooling_layer.cpp:129-318
def pool_forward(x, method, k, s, p):
    assert method in (0, 1), "method: 0 = MAX, 1 = AVE (PoolingParameter.PoolMethod)"
    N, C, H, W = x.shape
    Ho, Wo = pooled_extent(H, k[0], s[0], p[0]), pooled_extent(W, k[1], s[1], p[1])
    y = np.zeros((N, C, Ho, Wo), np.float32)
    mask = np.full((N, C, Ho, Wo), -1, np.int32)
    for ho in range(Ho):
        for wo in range(Wo):
            hs, ws = ho * s[0] - p[0], wo * s[1] - p[1]
            if method == 0:
                he, we = min(hs + k[0], H), min(ws + k[1], W)
                hs, ws = max(hs, 0), max(ws, 0)
                win = x[:, :, hs:he, ws:we].reshape(N, C, -1)
                idx = win.argmax(axis=2)                       # first maximum, like the strict '>' scan
                y[:, :, ho, wo] = np.take_along_axis(win, idx[..., None], 2)[..., 0]
                mask[:, :, ho, wo] = (hs + idx // (we - ws)) * W + (ws + idx % (we - ws))
            else:
                he, we = min(hs + k[0], H + p[0]), min(ws + k[1], W + p[1])
                size = (he - hs) * (we - ws)
                hs, ws, he, we = max(hs, 0), max(ws, 0), min(he, H), min(we, W)
                y[:, :, ho, wo] = x[:, :, hs:he, ws:we].sum(axis=(2, 3), dtype=np.float64) / size
    return y, mask


def pool_backward(dy, mask, x_shape, method, k, s, p):
    assert method in (0, 1)
    N, C, H, W = x_shape
    Ho, Wo = dy.shape[2:]
    dx = np.zeros(x_shape, np.float64)
    for ho in range(Ho):
        for wo in range(Wo):
            if method == 0:
                flat = dx.reshape(N, C, -1)
                np.add.at(flat, (np.arange(N)[:, None], np.arange(C)[None, :], mask[:, :, ho, wo]), dy[:, :, ho, wo])
            else:
                hs, ws = ho * s[0] - p[0], wo * s[1] - p[1]
                he, we = min(hs + k[0], H + p[0]), min(ws + k[1], W + p[1])
                size = (he - hs) * (we - ws)
                hs, ws, he, we = max(hs, 0), max(ws, 0), min(he, H), min(we, W)
                dx[:, :, hs:he, ws:we] += (dy[:, :, ho, wo] / size)[:, :, None, None]
    return dx.astype(np.float32)


# SoftmaxWithLossLayer::Forward_cpu / Backward_cpu, src/caffe/layers/softmax_loss_layer.cpp:96-160 (VALID normalisation)
def softmax_loss_forward(logits, labels):
    z = logits.astype(np.float64)
    z = z - z.max(axis=1, keepdims=True)
    p = np.exp(z)
    p /= p.sum(axis=1, keepdims=True)
    lab = labels.astype(np.int64)
    loss = -np.log(np.maximum(p[np.arange(len(lab)), lab], np.finfo(np.float32).tiny)).sum() / len(lab)
    return p.astype(np.float32), np.float32(loss)


def softmax_loss_backward(prob, labels, loss_weight=1.0):
    d = prob.astype(np.float64).copy()
    lab = labels.astype(np.int64)
    d[np.arange(len(lab)), lab] -= 1.0
    return (d * (loss_weight / len(lab))).astype(np.float32)


# InnerProductLayer::Forward_cpu / Backward_cpu, src/caffe/layers/inner_product_layer.cpp (transpose = false)
def ip_forward(x, w, b):
    y = x.reshape(x.shape[0], -1).astype(np.float64) @ w.astype(np.float64).T
    if b is not None:
        y += b
    return y.astype(np.float32)


def ip_backward(x, w, dy):
    x2 = x.reshape(x.shape[0], -1).astype(np.float64)
    dw = dy.astype(np.float64).T @ x2
    db = dy.astype(np.float64).sum(axis=0)
    dx = (dy.astype(np.float64) @ w.astype(np.float64)).reshape(x.shape)
    return dw.astype(np.float32), db.astype(np.float32), dx.astype(np.float32)


# InnerProductLayer::Backward_cpu's bias term (inner_product_layer.cpp, caffe_cpu_gemv of dy^T and the ones vector, beta = 1) and
# the convolution's backward_cpu_bias (base_conv_layer.cpp: one gemv per image): db0 + sum over images and pixels of dy[n][o][p]
def bias_backward(dy, db0):
    N, O = dy.shape[:2]
    return (db0.astype(np.float64) + dy.reshape(N, O, -1).astype(np.float64).sum(axis=(0, 2))).astype(np.float32)


# LRNLayer ACROSS_CHANNELS: CrossChannelForward_cpu / CrossChannelBackward_cpu, src/caffe/layers/lrn_layer.cpp; the forward
# is written the way the reference's own test states it (test_lrn_layer.cpp:61-91, ReferenceLRNForward, with k)
def lrn_forward(x, size=5, alpha=1.0, beta=0.75, k=1.0):
    N, C = x.shape[:2]
    x64 = x.astype(np.float64)
    scale = np.empty_like(x64)
    for c in range(C):
        lo_ = max(c - (size - 1) // 2, 0)
        hi_ = min(c - (size - 1) // 2 + size, C)
        scale[:, c] = k + (x64[:, lo_:hi_] ** 2).sum(axis=1) * alpha / size
    y = x64 * scale ** (-beta)
    return y.astype(np.float32), scale.astype(np.float32)


def lrn_backward(x, y, scale, dy, size=5, alpha=1.0, beta=0.75):
    C = x.shape[1]
    x64, y64, s64, d64 = (a.astype(np.float64) for a in (x, y, scale, dy))
    ratio = d64 * y64 / s64
    ipp = size - (size + 1) // 2                       # inverse_pre_pad
    dx = d64 * s64 ** (-beta)
    for c in range(C):
        lo_, hi_ = max(c - ipp, 0), min(c - ipp + size, C)
        dx[:, c] -= 2.0 * alpha * beta / size * x64[:, c] * ratio[:, lo_:hi_].sum(axis=1)
    return dx.astype(np.float32)


# DropoutLayer TRAIN, src/caffe/layers/dropout_layer.cpp: y = x * mask * 1/(1-ratio).  The mask generator is this
# repository's counter-based one (include/b2c.h b2c_dropout_mask): keep = (splitmix64(seed + offset + i) >> 40) >= ratio * 2^24
def dropout_mask(n, ratio, seed, offset=0):
    with np.errstate(over="ignore"):
        z = (np.uint64(seed) + np.uint64(offset) + np.arange(n, dtype=np.uint64)) + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    u = (z >> np.uint64(40)).astype(np.uint32)
    thr = np.uint32(int(float(np.float32(ratio)) * 16777216.0))
    return np.where(u >= thr, np.float32(1.0) / (np.float32(1.0) - np.float32(ratio)), np.float32(0.0)).astype(np.float32)


# AccuracyLayer::Forward_cpu, src/caffe/layers/accuracy_layer.cpp:44-100: partial_sort of (score, class) pairs with
# std::greater, the label must be among the first top_k; returns hits / N
def accuracy(scores, labels, top_k=1):
    hits = 0
    for i in range(scores.shape[0]):
        pairs = sorted(((float(v), j) for j, v in enumerate(scores[i])), reverse=True)
        hits += int(int(labels[i]) in [j for _, j in pairs[:top_k]])
    return np.float32(hits / scores.shape[0])


# DataTransformer<Dtype>::Transform(const Datum&, Dtype*, rand), src/caffe/data_transformer.cpp:178-312 (uint8 branch), batched:
# crop window + mirror per image, mean_value per channel or mean image in datum coordinates, scale
def transform_u8(src, crop, h_off, w_off, mirror, mean_values=None, mean_image=None, scale=1.0):
    N, Cc, Hd, Wd = src.shape
    ch, cw = crop
    out = np.empty((N, Cc, ch, cw), np.float32)
    for n in range(N):
        win = src[n, :, h_off[n]:h_off[n] + ch, w_off[n]:w_off[n] + cw].astype(np.float32)
        if mean_image is not None:
            win = win - mean_image[:, h_off[n]:h_off[n] + ch, w_off[n]:w_off[n] + cw].astype(np.float32)
        elif mean_values is not None:
            win = win - np.asarray(mean_values, np.float32).reshape(Cc, 1, 1)
        win = (win * np.float32(scale)).astype(np.float32)
        out[n] = win[:, :, ::-1] if mirror[n] else win
    return out

"""Float64 oracle of the transposed convolution (DeconvolutionLayer) and Crop, plus float32 restatements of the depthwise kernels.

Shapes follow the layer: x [N, C, H, W] (bottom), w [C, O/G, kh, kw], bias [O], y [N, O, Ht, Wt] with
Ht = sh*(H-1) + dh*(kh-1) + 1 - 2*ph (deconv_layer.cpp).  k, s, p, d are (h, w) pairs.

Two independent forward forms that must agree:
  * col2im form -- per image and group, col = W^T x (the reference's backward_gpu_gemm), then col2im scatters col onto the top;
  * gather form -- per output t and tap i, the bottom pixel h = (t + p - i*d) / s where that is an integer in range.
`phase_forward` restates the sub-pixel decomposition of the kernels' phase route in numpy.
"""
import math

import numpy as np


def out_extent(H, k, s, p, d):
    return s * (H - 1) + d * (k - 1) + 1 - 2 * p


def _pair(v):
    return tuple(v) if isinstance(v, (tuple, list)) else (v, v)


def deconv_forward_col2im(x, w, bias, k, s, p, d, G=1):
    x = np.asarray(x, np.float64); w = np.asarray(w, np.float64)
    (kh, kw), (sh, sw), (ph, pw), (dh, dw) = map(_pair, (k, s, p, d))
    N, C, H, W = x.shape
    Og = w.shape[1]; O = Og * G; Cg = C // G
    Ht, Wt = out_extent(H, kh, sh, ph, dh), out_extent(W, kw, sw, pw, dw)
    y = np.zeros((N, O, Ht, Wt))
    for n in range(N):
        for g in range(G):
            wg = w[g * Cg:(g + 1) * Cg].reshape(Cg, Og * kh * kw)                 # [Cg, (o, i, j)]
            col = (wg.T @ x[n, g * Cg:(g + 1) * Cg].reshape(Cg, H * W)).reshape(Og, kh, kw, H, W)
            for i in range(kh):
                for j in range(kw):
                    for h in range(H):
                        t = h * sh - ph + i * dh
                        if not 0 <= t < Ht:
                            continue
                        tw = np.arange(W) * sw - pw + j * dw
                        ok = (tw >= 0) & (tw < Wt)
                        row = y[n, g * Og:(g + 1) * Og, t]                           # a view [Og, Wt]
                        row[:, tw[ok]] += col[:, i, j, h, ok]
    if bias is not None:
        y += np.asarray(bias, np.float64)[None, :, None, None]
    return y


def _taps(T, H, k, s, p, d):
    """For each tap i: (t indices, h indices) of the outputs it reaches, gather form."""
    out = []
    t = np.arange(T)
    for i in range(k):
        num = t + p - i * d
        ok = (num >= 0) & (num % s == 0) & (num // s < H)
        out.append((t[ok], num[ok] // s))
    return out


def deconv_forward_gather(x, w, bias, k, s, p, d, G=1):
    x = np.asarray(x, np.float64); w = np.asarray(w, np.float64)
    (kh, kw), (sh, sw), (ph, pw), (dh, dw) = map(_pair, (k, s, p, d))
    N, C, H, W = x.shape
    Og = w.shape[1]; O = Og * G; Cg = C // G
    Ht, Wt = out_extent(H, kh, sh, ph, dh), out_extent(W, kw, sw, pw, dw)
    y = np.zeros((N, O, Ht, Wt))
    th, tw = _taps(Ht, H, kh, sh, ph, dh), _taps(Wt, W, kw, sw, pw, dw)
    for g in range(G):
        xg = x[:, g * Cg:(g + 1) * Cg]
        for i in range(kh):
            for j in range(kw):
                (ti, hi), (tj, wj) = th[i], tw[j]
                if not len(ti) or not len(tj):
                    continue
                xs = xg[:, :, hi][:, :, :, wj]                                      # [N, Cg, |ti|, |tj|]
                y[:, g * Og:(g + 1) * Og, ti[:, None], tj[None, :]] += np.einsum("nchw,co->nohw", xs, w[g * Cg:(g + 1) * Cg, :, i, j])
    if bias is not None:
        y += np.asarray(bias, np.float64)[None, :, None, None]
    return y


deconv_forward = deconv_forward_gather


def deconv_backward(x, w, dy, k, s, p, d, G=1):
    """(dx, dw, db) of y = deconv_forward(x, w, b): dx is the dual convolution's forward of dy."""
    x = np.asarray(x, np.float64); w = np.asarray(w, np.float64); dy = np.asarray(dy, np.float64)
    (kh, kw), (sh, sw), (ph, pw), (dh, dw_) = map(_pair, (k, s, p, d))
    N, C, H, W = x.shape
    Og = w.shape[1]; Cg = C // G
    Ht, Wt = dy.shape[2:]
    dx = np.zeros_like(x); dw = np.zeros_like(w)
    th, tw = _taps(Ht, H, kh, sh, ph, dh), _taps(Wt, W, kw, sw, pw, dw_)
    for g in range(G):
        for i in range(kh):
            for j in range(kw):
                (ti, hi), (tj, wj) = th[i], tw[j]
                if not len(ti) or not len(tj):
                    continue
                dys = dy[:, g * Og:(g + 1) * Og][:, :, ti][:, :, :, tj]             # [N, Og, |ti|, |tj|]
                xs = x[:, g * Cg:(g + 1) * Cg][:, :, hi][:, :, :, wj]
                dx[:, g * Cg:(g + 1) * Cg, hi[:, None], wj[None, :]] += np.einsum("nohw,co->nchw", dys, w[g * Cg:(g + 1) * Cg, :, i, j])
                dw[g * Cg:(g + 1) * Cg, :, i, j] += np.einsum("nchw,nohw->co", xs, dys)
    return dx, dw, dy.sum(axis=(0, 2, 3))


# ---- the phase decomposition, restated ----------------------------------------------------------------------------------
def phase_axis(t0, T, k, s, p, d):
    """(M, n, i0, L, dd, pad) of the outputs t0, t0 + s, ... < T: a stride-1 correlation of the bottom with the n taps
    i0 + (n-1-l)*L (l = 0..n-1), dilation dd, pad `pad`."""
    g = math.gcd(s, d)
    L, dd = s // g, d // g
    M = (T - t0 + s - 1) // s if t0 < T else 0
    r = (t0 + p) % s
    i0 = next((i for i in range(min(k, L)) if (i * d) % s == r), None)
    if i0 is None:
        return M, 0, 0, L, dd, 0
    n = (k - 1 - i0) // L + 1
    q0 = (i0 * d - r) // s
    return M, n, i0, L, dd, q0 + (n - 1) * dd - (t0 + p - r) // s


def phase_forward(x, w, bias, k, s, p, d, G=1):
    """The sub-pixel decomposition in float64: each of the sh*sw output phases as a stride-1 correlation with the flipped
    sub-filter, written onto its lattice of the top."""
    x = np.asarray(x, np.float64); w = np.asarray(w, np.float64)
    (kh, kw), (sh, sw), (ph, pw), (dh, dw) = map(_pair, (k, s, p, d))
    N, C, H, W = x.shape
    Og = w.shape[1]; O = Og * G; Cg = C // G
    Ht, Wt = out_extent(H, kh, sh, ph, dh), out_extent(W, kw, sw, pw, dw)
    y = np.full((N, O, Ht, Wt), np.nan)
    for t0h in range(sh):
        for t0w in range(sw):
            Mh, nh, i0h, Lh, ddh, padh = phase_axis(t0h, Ht, kh, sh, ph, dh)
            Mw, nw, i0w, Lw, ddw, padw = phase_axis(t0w, Wt, kw, sw, pw, dw)
            if not Mh or not Mw:
                continue
            out = np.zeros((N, O, Mh, Mw))
            for a in range(nh):
                for b in range(nw):
                    i = i0h + (nh - 1 - a) * Lh          # flipped sub-filter tap (a, b)
                    j = i0w + (nw - 1 - b) * Lw
                    hh = np.arange(Mh) - padh + a * ddh
                    ww = np.arange(Mw) - padw + b * ddw
                    okh, okw = (hh >= 0) & (hh < H), (ww >= 0) & (ww < W)
                    for g in range(G):
                        xs = x[:, g * Cg:(g + 1) * Cg][:, :, hh[okh]][:, :, :, ww[okw]]
                        out[:, g * Og:(g + 1) * Og, np.nonzero(okh)[0][:, None], np.nonzero(okw)[0][None, :]] += \
                            np.einsum("nchw,co->nohw", xs, w[g * Cg:(g + 1) * Cg, :, i, j])
            if bias is not None:
                out += np.asarray(bias, np.float64)[None, :, None, None]
            y[:, :, t0h::sh, t0w::sw] = out
    return y


# ---- float32 restatements of the depthwise kernels (deconv.cu), bit for bit ---------------------------------------------
def dw_forward_f32(x, w, bias, k, s, p, d):
    """deconv_dw_fwd_kernel: taps i ascending then j ascending, on-grid in-bounds only; fp32 product, then fp32 add, from +0;
    bias added last."""
    x = np.asarray(x, np.float32); w = np.asarray(w, np.float32)
    (kh, kw), (sh, sw), (ph, pw), (dh, dw) = map(_pair, (k, s, p, d))
    N, C, H, W = x.shape
    Ht, Wt = out_extent(H, kh, sh, ph, dh), out_extent(W, kw, sw, pw, dw)
    y = np.zeros((N, C, Ht, Wt), np.float32)
    th, tw = _taps(Ht, H, kh, sh, ph, dh), _taps(Wt, W, kw, sw, pw, dw)
    for i in range(kh):
        for j in range(kw):
            (ti, hi), (tj, wj) = th[i], tw[j]
            if not len(ti) or not len(tj):
                continue
            prod = (x[:, :, hi][:, :, :, wj] * w[None, :, 0, i, j, None, None]).astype(np.float32)
            idx = (slice(None), slice(None), ti[:, None], tj[None, :])
            y[idx] = (y[idx] + prod).astype(np.float32)
    if bias is not None:
        y = (y + np.asarray(bias, np.float32)[None, :, None, None]).astype(np.float32)
    return y


def dw_dgrad_f32(dy, w, H, W, k, s, p, d):
    """deconv_dw_dgrad_kernel: dx[h][w] = sum over taps i ascending then j ascending of dy[h*s - p + i*d][...] * w[i][j]."""
    dy = np.asarray(dy, np.float32); w = np.asarray(w, np.float32)
    (kh, kw), (sh, sw), (ph, pw), (dh, dw) = map(_pair, (k, s, p, d))
    N, C, Ht, Wt = dy.shape
    dx = np.zeros((N, C, H, W), np.float32)
    for i in range(kh):
        th = np.arange(H) * sh - ph + i * dh
        okh = (th >= 0) & (th < Ht)
        for j in range(kw):
            tw = np.arange(W) * sw - pw + j * dw
            okw = (tw >= 0) & (tw < Wt)
            if not okh.any() or not okw.any():
                continue
            prod = (dy[:, :, th[okh]][:, :, :, tw[okw]] * w[None, :, 0, i, j, None, None]).astype(np.float32)
            idx = (slice(None), slice(None), np.nonzero(okh)[0][:, None], np.nonzero(okw)[0][None, :])
            dx[idx] = (dx[idx] + prod).astype(np.float32)
    return dx


# ---- Crop (crop_layer.cpp) -----------------------------------------------------------------------------------------------
def crop_offsets(bottom_shape, ref_shape, axis=2, offset=()):
    """CropLayer::Reshape's rules: the top takes ref's extents from `axis` on (negative axes count from the end); one offset for
    all cropped axes or one per cropped axis; the window must fit.  Returns (top_shape, offsets over every axis); raises
    ValueError with the reference's message where it CHECK-fails."""
    nax = len(bottom_shape)
    if not -nax <= axis < nax:
        raise ValueError(f"axis {axis} out of range for final index {nax}")
    start = axis % nax
    if len(ref_shape) != nax:
        raise ValueError("Check failed: bottom[0]->num_axes() == bottom[1]->num_axes()")
    if len(offset) > 1 and len(offset) != nax - start:
        raise ValueError("number of offset values specified must be equal to the number of dimensions following axis.")
    top, offs = list(bottom_shape), [0] * nax
    for i in range(start, nax):
        o = 0 if not offset else offset[0] if len(offset) == 1 else offset[i - start]
        top[i] = ref_shape[i]
        if bottom_shape[i] - o < ref_shape[i]:
            raise ValueError(f"invalid crop parameters in dimension: {i}")
        offs[i] = o
    return tuple(top), tuple(offs)


def crop_forward(x, top_shape, offsets):
    return np.asarray(x)[tuple(slice(o, o + t) for o, t in zip(offsets, top_shape))].copy()


def crop_backward(dtop, bottom_shape, offsets):
    dx = np.zeros(bottom_shape, np.asarray(dtop).dtype)
    dx[tuple(slice(o, o + t) for o, t in zip(offsets, dtop.shape))] = dtop
    return dx


# ---- BilinearFiller (filler.hpp) ------------------------------------------------------------------------------------------
def bilinear_weights(shape):
    """The modelled reference's BilinearFiller: f = ceil(width / 2) with INTEGER division (so f = k // 2 for odd k, unlike
    BVLC's ceil(k / 2.)), c = (2f - 1 - f % 2) / (2f), w[x, y] = (1 - |x/f - c|) (1 - |y/f - c|) for every (num, channel)."""
    if len(shape) != 4:
        raise ValueError("Blob must be 4 dim.")
    if shape[2] != shape[3]:
        raise ValueError("Filter must be square")
    k = shape[3]
    f = int(math.ceil(k // 2))
    c = np.float32((2 * f - 1 - f % 2) / (2.0 * f))
    i = np.arange(int(np.prod(shape)))
    xx = (i % k).astype(np.float32)
    yy = ((i // k) % k).astype(np.float32)
    # x / f and the difference in float, 1. - |.| and the product in double, then stored as float
    ax = np.abs(xx / np.float32(f) - c).astype(np.float64)
    ay = np.abs(yy / np.float32(f) - c).astype(np.float64)
    return ((1.0 - ax) * (1.0 - ay)).astype(np.float32).reshape(shape)


# ---- a small encoder-decoder net through every new layer ----------------------------------------------------------------------
# data [N, 3, 8, 8] -> conv1 (6, 3x3/2 pad 1) -> [N, 6, 4, 4]
#   -> up  = Deconvolution (3, 4x4/2)                     -> [N, 3, 10, 10] -> crop (Crop to data, axis 2, offset 1) -> [N, 3, 8, 8]
#   -> bil = Deconvolution (6, 4x4/2 pad 1, group 6, bilinear, no bias, lr_mult 0: a frozen upsampler) -> [N, 6, 8, 8]
#      -> proj (Convolution 3, 1x1)                        -> [N, 3, 8, 8]
# sum = Eltwise SUM (crop, proj, data) -> SigmoidCrossEntropyLoss against target.
# Learnable blobs in layer order: conv1 w, b; up w, b; bil w; proj w, b.
def encdec_prototxt(N, force_nd=False, engine=""):
    nd = " force_nd_im2col: true" if force_nd else ""
    eng = f" engine: {engine}" if engine else ""
    return f'''name: "encdec"
layer {{ name: "data" type: "Input" top: "data" top: "target" input_param {{ shape {{ dim: {N} dim: 3 dim: 8 dim: 8 }} shape {{ dim: {N} dim: 192 }} }} }}
layer {{ name: "conv1" type: "Convolution" bottom: "data" top: "c1" convolution_param {{ num_output: 6 kernel_size: 3 stride: 2 pad: 1 }} }}
layer {{ name: "up" type: "Deconvolution" bottom: "c1" top: "up" convolution_param {{ num_output: 3 kernel_size: 4 stride: 2{nd}{eng} }} }}
layer {{ name: "crop" type: "Crop" bottom: "up" bottom: "data" top: "crop" crop_param {{ axis: 2 offset: 1 }} }}
layer {{ name: "bil" type: "Deconvolution" bottom: "c1" top: "bil" param {{ lr_mult: 0 decay_mult: 0 }}
  convolution_param {{ num_output: 6 kernel_size: 4 stride: 2 pad: 1 group: 6 bias_term: false weight_filler {{ type: "bilinear" }} }} }}
layer {{ name: "proj" type: "Convolution" bottom: "bil" top: "proj" convolution_param {{ num_output: 3 kernel_size: 1 }} }}
layer {{ name: "sum" type: "Eltwise" bottom: "crop" bottom: "proj" bottom: "data" top: "sum" }}
layer {{ name: "loss" type: "SigmoidCrossEntropyLoss" bottom: "sum" bottom: "target" top: "loss" }}
'''


def _conv(x, w, b, s, p):
    """float64 convolution (cross-correlation) and its backward, through the transposed-convolution oracle's tap tables."""
    x = np.asarray(x, np.float64); w = np.asarray(w, np.float64)
    N, C, H, W = x.shape
    O, _, k, _ = w.shape
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    y = np.zeros((N, O, Ho, Wo))
    for i in range(k):
        for j in range(k):
            h = np.arange(Ho) * s - p + i
            ww = np.arange(Wo) * s - p + j
            oh, ow = (h >= 0) & (h < H), (ww >= 0) & (ww < W)
            xs = x[:, :, h[oh]][:, :, :, ww[ow]]
            y[:, :, np.nonzero(oh)[0][:, None], np.nonzero(ow)[0][None, :]] += np.einsum("nchw,oc->nohw", xs, w[:, :, i, j])
    return y + np.asarray(b, np.float64)[None, :, None, None]


def _conv_back(x, w, dy, s, p):
    x = np.asarray(x, np.float64); w = np.asarray(w, np.float64)
    N, C, H, W = x.shape
    O, _, k, _ = w.shape
    Ho, Wo = dy.shape[2:]
    dx, dw = np.zeros_like(x), np.zeros_like(w)
    for i in range(k):
        for j in range(k):
            h = np.arange(Ho) * s - p + i
            ww = np.arange(Wo) * s - p + j
            oh, ow = (h >= 0) & (h < H), (ww >= 0) & (ww < W)
            hi, wi = h[oh], ww[ow]
            dys = dy[:, :, np.nonzero(oh)[0]][:, :, :, np.nonzero(ow)[0]]
            xs = x[:, :, hi][:, :, :, wi]
            dw[:, :, i, j] += np.einsum("nohw,nchw->oc", dys, xs)
            dx[:, :, hi[:, None], wi[None, :]] += np.einsum("nohw,oc->nchw", dys, w[:, :, i, j])
    return dx, dw, dy.sum(axis=(0, 2, 3))


def encdec_forward_backward(params, data, target):
    """(loss, [gradient of each learnable blob], blobs) of encdec_prototxt in float64; params in the net's learnable order."""
    w1, b1, wu, bu, wb, wp, bp = [np.asarray(a, np.float64) for a in params]
    N = data.shape[0]
    c1 = _conv(data, w1, b1, 2, 1)
    up = deconv_forward(c1, wu, bu, 4, 2, 0, 1)
    crop = up[:, :, 1:9, 1:9]
    bil = deconv_forward(c1, wb, None, 4, 2, 1, 1, G=6)
    proj = _conv(bil, wp, bp, 1, 0)
    x = crop + proj + np.asarray(data, np.float64)
    t = np.asarray(target, np.float64).reshape(x.shape)
    pos = (x >= 0).astype(np.float64)
    loss = -np.sum(x * (t - pos) - np.log1p(np.exp(x - 2 * x * pos))) / N
    dx = (1 / (1 + np.exp(-x)) - t) / N
    dbil, dwp, dbp = _conv_back(bil, wp, dx, 1, 0)
    dup = np.zeros_like(up); dup[:, :, 1:9, 1:9] = dx
    dc1u, dwu, dbu = deconv_backward(c1, wu, dup, 4, 2, 0, 1)
    dc1b, dwb, _ = deconv_backward(c1, wb, dbil, 4, 2, 1, 1, G=6)
    _, dw1, db1 = _conv_back(data, w1, dc1u + dc1b, 2, 1)
    return loss, [dw1, db1, dwu, dbu, dwb, dwp, dbp], dict(c1=c1, up=up, crop=crop, bil=bil, proj=proj, sum=x)

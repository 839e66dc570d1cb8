"""CPU tests of the oracle's restatements of the FFMA convolution kernels (b2o_conv_fwd_ffma / _dgrad_ffma / _wgrad_ffma in
oracle/b2o_oracle.c), the bit-exact yardstick tests/test_conv_ffma_schedule_gpu.py holds conv_simt.cu to.

Each restatement is pinned four ways: known answers on tiny shapes (the sign of an all-padding zero included), a derived bound
against the float64 oracle (b2o_conv_forward / b2o_conv_backward with acc64), equality with it on integer data, and sensitivity
to summation order, so that a bit-exact check against it would see a kernel that summed in another order.

The bounds.  Write u = 2^-24 and gamma_n = n u / (1 - n u).  A sum evaluated as a tree of depth n whose every node rounds once
(an fmaf rounds once; the first fmaf onto +0 is exact but is counted anyway) is off the exact sum by at most gamma_n times the
sum of the magnitudes of its terms (Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., 4.2).  The yardstick itself
rounds too, and its error adds:
  * forward: depth Kd taps + 1 for the bias.  The float64 leg rounds the tap sum to fp32 once (u |sum|) and the bias is added
    here in float64, so  |y - ref| <= (gamma_{Kd+1} + u) (sum |x w| + |b|).
  * data gradient: depth kh kw Og.  The float64 leg rounds each column entry to fp32 and sums up to kh kw of them in col2im's
    fp32 order, depth kh kw + 1:  |dx - ref| <= (gamma_{kh kw Og} + gamma_{kh kw + 1}) sum |dy w|.
  * weight gradient: depth ceil(N Ho Wo / 256) per thread + 5 butterfly levels + 8 warp partials + 1 add onto dw0.  The float64
    leg adds each image's float64 sum onto dw in fp32, N roundings:
    |dw - ref| <= (gamma_{ceil(Q/256) + 14} + gamma_N) (sum |dy x| + |dw0|).
The magnitudes come from the same oracle on |x|, |w|, |dy| (rounded to fp32 once: the factor 1 + 2^-20 covers that)."""
import numpy as np
import pytest

import oracle as o

U = 2.0 ** -24
SLACK = 1.0 + 2.0 ** -20


def gamma(n):
    return n * U / (1 - n * U)


def prm(N, C, H, W, O, k, s=1, p=0, d=1, G=1, bias=True):
    return o.ConvParams.make(N, C, H, W, O, k, s, p, d, G, bias)


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.int32)


def f64_dx(po, w, dy):
    return o.conv_backward(po, np.zeros(po.x_shape(), np.float32), w, dy, acc64=True)[2]


def f64_dw(po, x, dy, dw0):
    q = o.ConvParams.make(po.N, po.C, po.H, po.W, po.O, (po.kh, po.kw), (po.sh, po.sw), (po.ph, po.pw), (po.dh, po.dw), po.G, False)
    return o.conv_backward(q, x, np.zeros(po.w_shape(), np.float32), dy, dw=dw0, want_dx=False, acc64=True)[0]


# ---- known answers -------------------------------------------------------------------------------------------------------------
def test_fwd_known_answer_counts_inside_taps():
    po = prm(1, 1, 3, 3, 1, 3, p=1)
    y = o.conv_fwd_ffma(po, np.ones((1, 1, 3, 3), np.float32), np.ones((1, 1, 3, 3), np.float32), np.array([0.5], np.float32))
    assert np.array_equal(y[0, 0], np.array([[4.5, 6.5, 4.5], [6.5, 9.5, 6.5], [4.5, 6.5, 4.5]], np.float32))


def test_fwd_skips_padded_taps_and_adds_bias_last():
    """a 1x1 image under a 3x3 / pad 1 window: one inside tap.  Its product underflows to -0 and the eight padded taps are
    skipped, so -0 survives (multiplying them by 0 would give +0).  Products 1 then 2^24 with bias 1: the chain gives
    fl(1 + 2^24) = 2^24 (a tie, to even), then + 1 = 2^24 again; a chain started at the bias would give 2 + 2^24"""
    po = prm(1, 1, 1, 1, 1, 3, p=1, bias=False)
    w = np.zeros((1, 1, 3, 3), np.float32)
    w[0, 0, 1, 1] = 1e-30
    y = o.conv_fwd_ffma(po, np.full((1, 1, 1, 1), -1e-30, np.float32), w)
    assert bits(y)[0, 0, 0, 0] == bits(np.float32(-0.0))
    po = prm(1, 2, 1, 1, 1, 1)
    x = np.array([1.0, 4096.0], np.float32).reshape(1, 2, 1, 1)
    y = o.conv_fwd_ffma(po, x, x.reshape(1, 2, 1, 1), np.array([1.0], np.float32))
    assert y[0, 0, 0, 0] == np.float32(2.0 ** 24)


def test_fwd_all_padding_output_is_plus_zero_or_bias():
    po = prm(1, 2, 2, 2, 3, 3, p=4, bias=False)          # pad >= k: the corner outputs see only padding
    x = np.full(po.x_shape(), -1.0, np.float32)
    w = np.full(po.w_shape(), 1.0, np.float32)
    y = o.conv_fwd_ffma(po, x, w)
    assert bits(y)[0, 0, 0, 0] == 0 and y[0, 0, 0, 0] == 0.0
    b = np.array([-0.5, 0.0, 2.0], np.float32)
    yb = o.conv_fwd_ffma(prm(1, 2, 2, 2, 3, 3, p=4), x, w, b)
    assert np.array_equal(yb[0, :, 0, 0], b)


def test_dgrad_known_answer_strided_grid():
    """3x3 / stride 2 / pad 0 on 5x5: a dx pixel gets one tap per (ho, wo) whose window covers it; per axis 1, 1, 2, 1, 1"""
    po = prm(1, 1, 5, 5, 1, 3, s=2, bias=False)
    dx = o.conv_dgrad_ffma(po, np.ones(po.w_shape(), np.float32), np.ones(po.y_shape(), np.float32))
    per = np.array([1, 1, 2, 1, 1], np.float32)
    assert np.array_equal(dx[0, 0], np.outer(per, per))


def test_dgrad_known_answer_groups():
    """G = 2: dx of group g sums only that group's outputs"""
    po = prm(1, 4, 3, 3, 6, 1, G=2, bias=False)
    w = np.arange(1, 1 + 6 * 2, dtype=np.float32).reshape(6, 2, 1, 1)
    dy = np.ones(po.y_shape(), np.float32)
    dx = o.conv_dgrad_ffma(po, w, dy)
    want = [w[0:3, 0].sum(), w[0:3, 1].sum(), w[3:6, 0].sum(), w[3:6, 1].sum()]
    assert np.array_equal(dx[0, :, 1, 1], np.array(want, np.float32))


def test_wgrad_known_answer_accumulates_onto_dw0():
    po = prm(2, 1, 3, 3, 1, 3, p=1, bias=False)
    dw0 = np.full(po.w_shape(), 0.25, np.float32)
    dw = o.conv_wgrad_ffma(po, np.ones(po.x_shape(), np.float32), np.ones(po.y_shape(), np.float32), dw0)
    cnt = np.array([[4, 6, 4], [6, 9, 6], [4, 6, 4]], np.float32) * 2
    assert np.array_equal(dw[0, 0], cnt + 0.25)
    assert np.array_equal(o.conv_wgrad_ffma(po, np.ones(po.x_shape(), np.float32), np.ones(po.y_shape(), np.float32))[0, 0], cnt)


# ---- float64 bound and integer equality ----------------------------------------------------------------------------------------
SHAPES = [
    ("3x3_p1", dict(N=2, C=5, H=9, W=11, O=4, k=3, p=1)),
    ("7x7_s2_p3", dict(N=1, C=3, H=23, W=23, O=8, k=7, s=2, p=3)),
    ("g3_dil2", dict(N=2, C=6, H=12, W=12, O=9, k=3, p=2, d=2, G=3)),
    ("rect_s2x3_pad_ge_k", dict(N=3, C=4, H=8, W=13, O=5, k=(1, 3), s=(2, 3), p=(1, 3))),
    ("wide_q_1x1_s2", dict(N=5, C=16, H=25, W=23, O=7, k=1, s=2)),
]
SIDS = [s[0] for s in SHAPES]


def make_prm(c, bias=True):
    c = dict(c)
    return prm(c.pop("N"), c.pop("C"), c.pop("H"), c.pop("W"), c.pop("O"), c.pop("k"), bias=bias, **c)


@pytest.mark.parametrize("sid,c", SHAPES, ids=SIDS)
def test_restatements_within_float64_bound(rng, sid, c):
    po = make_prm(c)
    x = rng.standard_normal(po.x_shape()).astype(np.float32)
    w = rng.standard_normal(po.w_shape()).astype(np.float32)
    b = rng.standard_normal(po.O).astype(np.float32)
    dy = rng.standard_normal(po.y_shape()).astype(np.float32)
    dw0 = rng.standard_normal(po.w_shape()).astype(np.float32)
    nob = make_prm(c, bias=False)
    ax, aw, ady = np.abs(x), np.abs(w), np.abs(dy)
    # forward
    ref = o.conv_forward(nob, x, w, acc64=True).astype(np.float64) + b[None, :, None, None]
    mag = o.conv_forward(nob, ax, aw, acc64=True).astype(np.float64) * SLACK + np.abs(b)[None, :, None, None]
    y = o.conv_fwd_ffma(po, x, w, b)
    assert (np.abs(y - ref) <= (gamma(po.Kd + 1) + U) * mag).all()
    # data gradient
    taps = po.kh * po.kw
    ref = f64_dx(nob, w, dy).astype(np.float64)
    mag = f64_dx(nob, aw, ady).astype(np.float64) * SLACK
    dx = o.conv_dgrad_ffma(po, w, dy)
    assert (np.abs(dx - ref) <= (gamma(taps * (po.O // po.G)) + gamma(taps + 1)) * mag).all()
    # weight gradient
    Q = po.N * po.Ho * po.Wo
    ref = f64_dw(nob, x, dy, dw0).astype(np.float64)
    mag = f64_dw(nob, ax, ady, np.abs(dw0)).astype(np.float64) * SLACK
    dw = o.conv_wgrad_ffma(po, x, dy, dw0)
    assert (np.abs(dw - ref) <= (gamma(-(-Q // 256) + 14) + gamma(po.N)) * mag).all()


@pytest.mark.parametrize("sid,c", SHAPES, ids=SIDS)
def test_restatements_equal_float64_on_integers(rng, sid, c):
    """integers in [-4, 4]: every partial sum is an integer below 2^24, exact in any order"""
    po, nob = make_prm(c), make_prm(c, bias=False)

    def ints(shp):
        return rng.integers(-4, 5, shp).astype(np.float32)

    x, w, b, dy, dw0 = ints(po.x_shape()), ints(po.w_shape()), ints(po.O), ints(po.y_shape()), ints(po.w_shape())
    assert np.array_equal(o.conv_fwd_ffma(po, x, w, b), o.conv_forward(po, x, w, b, acc64=True))
    assert np.array_equal(o.conv_dgrad_ffma(po, w, dy), f64_dx(nob, w, dy))
    assert np.array_equal(o.conv_wgrad_ffma(po, x, dy, dw0), f64_dw(nob, x, dy, dw0))


# ---- order sensitivity ---------------------------------------------------------------------------------------------------------
def test_restatements_are_order_sensitive(rng):
    """the same sums with one loop's order reversed (channels for the forward, the outputs of the group for the data gradient,
    the images -- so each thread's chain and the warp partials change -- for the weight gradient) give different bits on most
    elements: a kernel that summed in another order would fail a bit-exact check against these restatements"""
    po = prm(4, 16, 12, 12, 16, 3, p=1)                   # Q = 576: three chunks of 256
    x = rng.standard_normal(po.x_shape()).astype(np.float32)
    w = rng.standard_normal(po.w_shape()).astype(np.float32)
    dy = rng.standard_normal(po.y_shape()).astype(np.float32)
    y = o.conv_fwd_ffma(po, x, w)
    y_rev = o.conv_fwd_ffma(po, x[:, ::-1], w[:, ::-1])
    assert np.mean(bits(y) != bits(y_rev)) > 0.5
    dx = o.conv_dgrad_ffma(po, w, dy)
    dx_rev = o.conv_dgrad_ffma(po, w[::-1], dy[:, ::-1])
    assert np.mean(bits(dx) != bits(dx_rev)) > 0.5
    dw = o.conv_wgrad_ffma(po, x, dy)
    dw_rev = o.conv_wgrad_ffma(po, x[::-1], dy[::-1])
    assert np.mean(bits(dw) != bits(dw_rev)) > 0.5
    # nor is any of them the im2col + GEMM order of the fp32 oracle (padded taps multiplied in, a plain a*b + acc)
    assert np.mean(bits(y) != bits(o.conv_forward(po, x, w, acc64=False))) > 0.3

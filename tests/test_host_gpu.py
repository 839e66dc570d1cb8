"""GPU tests of the C++ host layer: caffe::ConvolutionLayer created through LayerRegistry, driven through
SetUp / Forward / Backward like the reference's test_convolution_layer.cpp, and SGDSolver + ReduceScheduler
through several iterations like test_gradient_based_solver.cpp -- all checked against the CPU oracle."""
import numpy as np
import pytest

import oracle as o
from cases import EDGE_CASES, MODEL_CASES, REF_TEST_CASES, make, tensors, rel_err

pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from caffe_mpi_b200 import capi, host_api as h  # noqa: E402

SOME = REF_TEST_CASES + EDGE_CASES[:6] + [MODEL_CASES[i] for i in (0, 2, 5, 7, 9)]


@pytest.mark.parametrize("engine", [capi.ENGINE_DEFAULT, capi.ENGINE_CAFFE], ids=["default", "caffe"])
@pytest.mark.parametrize("name,case", SOME, ids=[c[0] for c in SOME])
def test_convolution_layer_forward_backward(rng, name, case, engine):
    po = make(o, case)
    x, w, b, dy = tensors(rng, po)
    L = h.ConvolutionLayer(po.O, (po.kh, po.kw), (po.sh, po.sw), (po.ph, po.pw), (po.dh, po.dw), po.G, bool(po.has_bias), engine)
    assert L.setup(po.x_shape()) == po.y_shape()               # TestSetup :190
    assert L.num_blobs() == 1 + po.has_bias
    L.set_blob(0, w)
    if po.has_bias:
        L.set_blob(1, b)
    y = L.forward(x)
    assert rel_err(y, o.conv_forward(po, x, w, b, acc64=True)) < 1e-4
    dx = L.backward(dy)
    dw_ref, db_ref, dx_ref = o.conv_backward(po, x, w, dy, acc64=True)
    assert rel_err(dx, dx_ref) < 1e-4
    assert rel_err(L.get_blob(0, diff=True).reshape(po.w_shape()), dw_ref) < 1e-4
    if po.has_bias:
        assert rel_err(L.get_blob(1, diff=True), db_ref) < 1e-4
    # param diffs accumulate across Backward calls (GradientChecker relies on it), bottom diff is overwritten
    dx2 = L.backward(dy)
    assert np.array_equal(dx, dx2)
    assert rel_err(L.get_blob(0, diff=True).reshape(po.w_shape()), 2 * dw_ref) < 1e-4


def nd_conv_oracle(x, w, b, k, s, p, d):
    """N-D conv forward from the oracle's im2col_nd + GEMM (base_conv_layer.hpp:36-60 with the N-D im2col)."""
    N, O = x.shape[0], w.shape[0]
    outs = []
    for n in range(N):
        col = o.im2col_nd(x[n], k, s, p, d)
        P = int(np.prod(col.shape[1:]))
        y = o.gemm(0, 0, O, P, col.shape[0], 1.0, w.reshape(O, -1), col.reshape(col.shape[0], P), 0.0, np.zeros((O, P), np.float32), acc64=True)
        if b is not None:
            y = y + b[:, None]
        outs.append(y.reshape((O,) + col.shape[1:]))
    return np.stack(outs)


def test_3d_convolution_nd_path(rng):
    # TestSimple3DConvolution :352 -- 3 spatial axes go through im2col_nd + GEMM
    x = rng.standard_normal((2, 3, 5, 6, 4)).astype(np.float32)
    w = rng.standard_normal((4, 3, 3, 2, 3)).astype(np.float32) * 0.2
    b = rng.standard_normal(4).astype(np.float32)
    k, s, p, d = (3, 2, 3), (2, 1, 1), (1, 0, 1), (1, 2, 1)
    L = h.ConvolutionLayer(4, k, s, p, d, 1, True)
    L.setup(x.shape)
    L.set_blob(0, w)
    L.set_blob(1, b)
    want = nd_conv_oracle(x, w, b, k, s, p, d)
    assert L.top_shape == want.shape
    assert rel_err(L.forward(x), want) < 2e-5
    # backward of the N-D path against finite differences of the oracle forward on a few coordinates
    dy = rng.standard_normal(want.shape).astype(np.float32)
    dx = L.backward(dy)
    for idx in rng.choice(x.size, 6, replace=False):
        xp, xm = x.copy().reshape(-1), x.copy().reshape(-1)
        xp[idx] += 1e-2
        xm[idx] -= 1e-2
        est = float(((nd_conv_oracle(xp.reshape(x.shape), w, b, k, s, p, d).astype(np.float64) -
                      nd_conv_oracle(xm.reshape(x.shape), w, b, k, s, p, d)) * dy).sum() / 2e-2)
        assert abs(est - dx.reshape(-1)[idx]) <= 1e-3 * max(1.0, abs(est))


def test_force_nd_im2col_equals_2d_path(rng):
    """TestNDAgainst2D :606.  y, dx and dW are the same bits: both paths issue the same GEMM calls at the same offsets (the bias
    as a K = 1 GEMM, fl(bias + y), against the bias kernel's fl(y + bias)), and col2im_nd sums in col2im's ascending (i, j)
    order.  db is reduced in different orders (bias_grad_kernel against a GEMV per image): each is within gamma_{N P} sum |dy|
    of the exact sum, so they differ by at most twice that."""
    po = o.ConvParams.make(2, 4, 9, 7, 5, 3, 2, 1, 1, 1, True)
    x, w, b, dy = tensors(rng, po)
    outs = []
    for force in (False, True):
        L = h.ConvolutionLayer(po.O, 3, 2, 1, 1, 1, True, capi.ENGINE_CAFFE, force_nd=force)
        L.setup(po.x_shape())
        L.set_blob(0, w)
        L.set_blob(1, b)
        y = L.forward(x)
        dx = L.backward(dy)
        outs.append((y, dx, L.get_blob(0, True), L.get_blob(1, True)))
    for name, a, c in zip(("y", "dx", "dW"), outs[0][:3], outs[1][:3]):
        assert np.array_equal(a.view(np.int32), c.view(np.int32)), name
    n = po.N * po.Ho * po.Wo
    bound = 2 * n * 2.0 ** -24 / (1 - n * 2.0 ** -24) * np.abs(dy).sum((0, 2, 3))
    assert (np.abs(outs[0][3].astype(np.float64) - outs[1][3]) <= bound).all()


def test_wrong_weight_shape_is_fatal():
    L = h.ConvolutionLayer(4, 3)
    with pytest.raises(h.HostError, match="kernel larger than padded input|Check failed"):
        L.setup((1, 3, 2, 2))


@pytest.mark.parametrize("policy", [dict(lr_policy="fixed"), dict(lr_policy="poly", power=2.0, max_iter=100),
                                    dict(lr_policy="step", gamma=0.5, stepsize=2)])
def test_sgd_solver_iterations_match_oracle(rng, policy):
    """K iterations of momentum SGD with weight decay, per-param lr_mult/decay_mult, on a 5-blob arena with odd
    sizes (even-padded slots): the (K+1)-th state equals the oracle's closed form applied K times
    (test_gradient_based_solver.cpp:228-414)."""
    counts = [7, 1024, 3, 50001, 12]
    lr_mult = [1.0, 2.0, 1.0, 0.5, 0.0]
    dc_mult = [1.0, 0.0, 1.0, 1.0, 1.0]
    cfg = dict(base_lr=0.05, momentum=0.9, weight_decay=0.004, **policy)
    s = h.SGDSolver(**cfg)
    s.set_params(counts, lr_mult, dc_mult)
    w = [rng.standard_normal(c).astype(np.float32) for c in counts]
    hist = [np.zeros(c, np.float32) for c in counts]
    for i, a in enumerate(w):
        s.set(i, a)
    for it in range(4):
        g = [rng.standard_normal(c).astype(np.float32) for c in counts]
        for i, a in enumerate(g):
            s.set(i, a, diff=True)
        lr = o.learning_rate(cfg["lr_policy"], it, cfg["base_lr"], cfg.get("gamma", 0.1), cfg.get("power", 1.0),
                             cfg.get("stepsize", 1), cfg.get("max_iter", 1))
        s.step()
        assert s.iter() == it + 1
        for i in range(len(counts)):
            _, w[i], hist[i] = o.sgd_update(g[i], w[i], hist[i], 0.9, lr * lr_mult[i], 0.004 * dc_mult[i])
            assert np.allclose(s.get(i, 0), w[i], rtol=2e-5, atol=2e-6)
            assert np.allclose(s.get(i, 2), hist[i], rtol=2e-5, atol=2e-6)
            assert np.array_equal(s.get(i, 1), np.zeros(counts[i], np.float32))     # diffs cleared by the update

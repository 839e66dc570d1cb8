"""GPU parity tests of the non-convolution layer kernels (csrc/layers.cu) through the C ABI against
oracle/layers_oracle.py.  Tolerance: fp32 elementwise / reduction work, 1e-5 relative (blob level)."""
import ctypes as C

import numpy as np
import pytest

from oracle import layers_oracle as lo
from cases import rel_err

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import caffe_mpi_b200 as m  # noqa: E402
from caffe_mpi_b200 import capi  # noqa: E402

TOL = 2e-5


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


def p(t):
    return C.c_void_p(t.data_ptr())


def st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def test_relu(rng):
    for n in (1, 5, 1000, 4097):
        x = rng.standard_normal(n).astype(np.float32)
        dy = rng.standard_normal(n).astype(np.float32)
        X, DY = dev(x), dev(dy)
        Y, DX = torch.empty_like(X), torch.empty_like(X)
        capi.check(m.lib().b2c_relu_forward(n, p(X), p(Y), 0.0, st()))
        capi.check(m.lib().b2c_relu_backward(n, p(DY), p(X), p(DX), 0.0, st()))
        assert np.array_equal(host(Y), lo.relu_forward(x)) and np.array_equal(host(DX), lo.relu_backward(dy, x))
        capi.check(m.lib().b2c_relu_forward(n, p(X), p(X), 0.0, st()))      # in place, like the prototxt uses it
        assert np.array_equal(host(X), lo.relu_forward(x))


@pytest.mark.parametrize("shape", [(4, 3, 5, 5), (8, 64, 14, 14), (2, 256, 7, 7), (3, 5, 1, 1)])
def test_batchnorm_train(rng, shape):
    N, Cc, H, W = shape
    S = H * W
    x = (rng.standard_normal(shape) * 1.5 + 0.3).astype(np.float32)
    g, b = rng.standard_normal(Cc).astype(np.float32), rng.standard_normal(Cc).astype(np.float32)
    dy = rng.standard_normal(shape).astype(np.float32)
    rm, rv = np.zeros(Cc, np.float32), np.zeros(Cc, np.float32)
    X, G, B, DY = dev(x), dev(g), dev(b), dev(dy)
    RM, RV = dev(rm), dev(rv)
    SM, SI = torch.empty(Cc, device="cuda"), torch.empty(Cc, device="cuda")
    XN, Y = torch.empty_like(X), torch.empty_like(X)
    for it, first in ((0, 1), (1, 0)):
        want = lo.bn_forward_train(x, g, b, 1e-4, 0.9, rm, rv, bool(first))
        capi.check(m.lib().b2c_bn_forward_train(N, Cc, S, p(X), p(G), p(B), 1e-4, 0.9, first, p(RM), p(RV), p(SM), p(SI), p(XN), p(Y), st()))
        y, xn, mean, invstd, rm, rv = want
        assert rel_err(host(Y), y) < TOL and rel_err(host(XN), xn) < TOL
        assert np.allclose(host(RM), rm, rtol=1e-5, atol=1e-6) and np.allclose(host(RV), rv, rtol=1e-5, atol=1e-6)
    DG, DB, DX = torch.full((Cc,), 9.0, device="cuda"), torch.full((Cc,), 9.0, device="cuda"), torch.empty_like(X)
    capi.check(m.lib().b2c_bn_backward(N, Cc, S, p(DY), p(XN), p(G), p(SI), p(DG), p(DB), p(DX), st()))
    dg, db, dx = lo.bn_backward(dy, xn, g, invstd)
    assert rel_err(host(DG), dg) < TOL and rel_err(host(DB), db) < TOL and rel_err(host(DX), dx) < 5e-5   # overwritten, not += 9


@pytest.mark.parametrize("relu", [0, 1])
@pytest.mark.parametrize("shape", [(4, 3, 5, 5), (8, 64, 14, 14), (2, 256, 7, 7), (3, 5, 1, 1), (8, 16, 64, 64), (64, 64, 56, 56), (37, 40, 30, 30)])
def test_batchnorm_fused_is_bitwise_the_unfused_chain(rng, shape, relu):
    """b2c_bn_forward_train_fused / b2c_bn_backward_fused (one launch each: cluster reduction + elementwise walk of the same slice)
    against BatchNorm [+ ReLU] run as separate layers: same bits for y, the saved and running statistics, dgamma, dbeta and dx.
    Shapes cover one CTA per channel, clusters of 2..8, float4 and scalar planes, slices that end inside a plane."""
    N, Cc, H, W = shape
    S = H * W
    L = m.lib()
    X = dev((rng.standard_normal(shape) * 1.5 + 0.3).astype(np.float32))
    G, B = dev(rng.standard_normal(Cc).astype(np.float32)), dev(rng.standard_normal(Cc).astype(np.float32))
    DY = dev(rng.standard_normal(shape).astype(np.float32))
    out = []
    for fused in (0, 1):
        RM, RV = torch.zeros(Cc, device="cuda"), torch.zeros(Cc, device="cuda")
        SM, SI = torch.empty(Cc, device="cuda"), torch.empty(Cc, device="cuda")
        Y, DX = torch.empty_like(X), torch.empty_like(X)
        DG, DB = torch.full((Cc,), 9.0, device="cuda"), torch.full((Cc,), 9.0, device="cuda")
        for first in (1, 0):
            if fused:
                capi.check(L.b2c_bn_forward_train_fused(N, Cc, S, p(X), p(G), p(B), 1e-4, 0.9, first, p(RM), p(RV), p(SM), p(SI), p(Y), relu, st()))
            else:
                XN = torch.empty_like(X)
                capi.check(L.b2c_bn_forward_train(N, Cc, S, p(X), p(G), p(B), 1e-4, 0.9, first, p(RM), p(RV), p(SM), p(SI), p(XN), p(Y), st()))
                if relu:
                    capi.check(L.b2c_relu_forward(X.numel(), p(Y), p(Y), 0.0, st()))
        if fused:
            capi.check(L.b2c_bn_backward_fused(N, Cc, S, p(DY), p(X), p(SM), p(SI), p(G), p(B), p(DG), p(DB), p(DX), relu, st()))
        else:
            D = DY
            if relu:
                D = torch.empty_like(DY)
                capi.check(L.b2c_relu_backward(X.numel(), p(DY), p(Y), p(D), 0.0, st()))
            capi.check(L.b2c_bn_backward(N, Cc, S, p(D), p(XN), p(G), p(SI), p(DG), p(DB), p(DX), st()))
        out.append([host(t) for t in (Y, SM, SI, RM, RV, DG, DB, DX)])
    for name, a, b in zip(("y", "mean", "invstd", "run_mean", "run_var", "dgamma", "dbeta", "dx"), out[0], out[1]):
        assert np.array_equal(a, b), name


@pytest.mark.parametrize("two_parts", [False, True], ids=["one_diff", "split_diff"])
@pytest.mark.parametrize("shape", [(4, 3, 5, 5), (8, 64, 14, 14), (2, 256, 7, 7), (8, 16, 64, 64), (64, 256, 56, 56), (37, 40, 30, 30)])
def test_batchnorm_residual_tail_is_bitwise_the_three_layers(rng, shape, two_parts):
    """b2c_bn_forward_train_fused_res / b2c_bn_backward_fused_res (BatchNorm -> Eltwise SUM -> in-place ReLU as one launch each way)
    against the three layers run one after the other: same bits for the sum's top, the statistics, dgamma, dbeta, the BatchNorm
    bottom diff and the diff handed to the sum's other bottom.  split_diff: the sum's top diff arrives in two parts (a blob with two
    consumers) -- the fused backward adds them on the fly, the unfused chain with b2c_add first."""
    N, Cc, H, W = shape
    S = H * W
    L = m.lib()
    X = dev((rng.standard_normal(shape) * 1.5 + 0.3).astype(np.float32))
    R = dev(rng.standard_normal(shape).astype(np.float32))
    G, B = dev(rng.standard_normal(Cc).astype(np.float32)), dev(rng.standard_normal(Cc).astype(np.float32))
    DS = dev(rng.standard_normal(shape).astype(np.float32))
    DS2 = dev(rng.standard_normal(shape).astype(np.float32)) if two_parts else None
    out = []
    for fused in (0, 1):
        RM, RV = torch.zeros(Cc, device="cuda"), torch.zeros(Cc, device="cuda")
        SM, SI = torch.empty(Cc, device="cuda"), torch.empty(Cc, device="cuda")
        YS, DX, DR = torch.empty_like(X), torch.empty_like(X), torch.empty_like(X)
        DG, DB = torch.full((Cc,), 9.0, device="cuda"), torch.full((Cc,), 9.0, device="cuda")
        if fused:
            capi.check(L.b2c_bn_forward_train_fused_res(N, Cc, S, p(X), p(G), p(B), 1e-4, 0.9, 1, p(RM), p(RV), p(SM), p(SI), p(R), p(YS), 1, st()))
            capi.check(L.b2c_bn_backward_fused_res(N, Cc, S, p(DS), p(DS2) if two_parts else None, p(YS), p(X), p(SM), p(SI), p(G), p(B), p(DG), p(DB),
                                                   p(DX), p(DR), st()))
        else:
            XN, YB, DA = torch.empty_like(X), torch.empty_like(X), torch.empty_like(X)
            capi.check(L.b2c_bn_forward_train(N, Cc, S, p(X), p(G), p(B), 1e-4, 0.9, 1, p(RM), p(RV), p(SM), p(SI), p(XN), p(YB), st()))
            capi.check(L.b2c_add_relu(X.numel(), p(YB), p(R), p(YS), st()))
            DT = DS
            if two_parts:
                DT = torch.empty_like(DS)
                capi.check(L.b2c_add(X.numel(), p(DS), p(DS2), p(DT), st()))
            capi.check(L.b2c_relu_backward2(X.numel(), p(DT), p(YS), p(DA), p(DR), st()))
            capi.check(L.b2c_bn_backward(N, Cc, S, p(DA), p(XN), p(G), p(SI), p(DG), p(DB), p(DX), st()))
        out.append([host(t) for t in (YS, SM, SI, RM, RV, DG, DB, DX, DR)])
    for name, a, b in zip(("y_sum", "mean", "invstd", "run_mean", "run_var", "dgamma", "dbeta", "dx", "d_residual"), out[0], out[1]):
        assert np.array_equal(a, b), name


def test_add_and_bias(rng):
    a, b = rng.standard_normal(1001).astype(np.float32), rng.standard_normal(1001).astype(np.float32)
    A, B = dev(a), dev(b)
    Y = torch.empty_like(A)
    capi.check(m.lib().b2c_add(1001, p(A), p(B), p(Y), st()))
    assert np.array_equal(host(Y), a + b)
    y = rng.standard_normal((4, 10)).astype(np.float32)
    bias = rng.standard_normal(10).astype(np.float32)
    Yv, Bv = dev(y.copy()), dev(bias)
    capi.check(m.lib().b2c_bias_forward(4, 10, 1, p(Bv), p(Yv), st()))
    assert np.allclose(host(Yv), y + bias, atol=1e-6)
    DB = dev(np.ones(10, np.float32))
    capi.check(m.lib().b2c_bias_backward(4, 10, 1, p(dev(y)), p(DB), st()))
    assert np.allclose(host(DB), 1 + y.sum(0), atol=1e-5)


@pytest.mark.parametrize("N,Cc", [(5, 7), (64, 1000), (3, 10)])
def test_softmax_loss(rng, N, Cc):
    z = (rng.standard_normal((N, Cc)) * 3).astype(np.float32)
    lab = rng.integers(0, Cc, N).astype(np.float32)
    Z, L = dev(z), dev(lab)
    P = torch.empty((N, Cc), device="cuda")
    loss = torch.empty(1, device="cuda")
    DX = torch.empty((N, Cc), device="cuda")
    capi.check(m.lib().b2c_softmax_loss_forward(N, Cc, p(Z), p(L), p(P), p(loss), st()))
    capi.check(m.lib().b2c_softmax_loss_backward(N, Cc, p(P), p(L), 1.0, p(DX), st()))
    pr, lo_ = lo.softmax_loss_forward(z, lab)
    assert rel_err(host(P), pr) < TOL and abs(float(host(loss)[0]) - float(lo_)) < 1e-5 * max(1.0, abs(float(lo_)))
    assert rel_err(host(DX), lo.softmax_loss_backward(pr, lab)) < TOL

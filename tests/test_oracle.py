"""CPU tests: pin the oracle (oracle/b2o_oracle.c) against the reference's own known-answer vectors,
against oracle/_ref (the reference's im2col.cpp compiled verbatim) and against the committed golden
fixtures.  No GPU needed."""
import os

import numpy as np
import pytest

import oracle as o
from cases import ALL_CASES, REF_TEST_CASES, make, tensors, rel_err

GOLD = os.path.join(os.path.dirname(__file__), "golden")


# ---- test_util_blas.cpp:19-175 integer known answers (EXPECT_EQ -> exact) -----------------------
def test_gemm_known_answers():
    data = np.arange(1, 13, dtype=np.float32)
    A, B = data[:6], data
    At = np.array([1, 4, 2, 5, 3, 6], np.float32)
    Bt = np.array([1, 5, 9, 2, 6, 10, 3, 7, 11, 4, 8, 12], np.float32)
    want = np.array([38, 44, 50, 56, 83, 98, 113, 128], np.float32)
    z = np.zeros(8, np.float32)
    for acc64 in (False, True):
        assert np.array_equal(o.gemm(0, 0, 2, 4, 3, 1.0, A, B, 0.0, z, acc64), want)
        assert np.array_equal(o.gemm(1, 0, 2, 4, 3, 1.0, At, B, 0.0, z, acc64), want)
        assert np.array_equal(o.gemm(1, 1, 2, 4, 3, 1.0, At, Bt, 0.0, z, acc64), want)
        assert np.array_equal(o.gemm(0, 1, 2, 4, 3, 1.0, A, Bt, 0.0, z, acc64), want)


def test_gemm_beta1_known_answer():
    A = np.array([1, 2, 3, 4, 5, 6], np.float32)
    B = np.array([1, 2], np.float32)
    res = np.array([5, 11, 17], np.float32)
    assert np.array_equal(o.gemm(0, 0, 3, 1, 2, 1.0, A, B, 1.0, res), res * 2)


def test_gemv_known_answers():
    A = np.arange(1, 7, dtype=np.float32)
    assert np.array_equal(o.gemv(0, 2, 3, 1.0, A, A[:3], 0.0, np.zeros(2, np.float32)), [14, 32])
    assert np.array_equal(o.gemv(1, 2, 3, 1.0, A, A[:2], 0.0, np.zeros(3, np.float32)), [9, 12, 15])
    assert np.array_equal(o.gemv(0, 3, 2, 1.0, A, A[:2], 0.0, np.zeros(3, np.float32)), [5, 11, 17])
    assert np.array_equal(o.gemv(1, 3, 2, 1.0, A, A[:3], 0.0, np.zeros(2, np.float32)), [22, 28])


# ---- FFMA emulators (b2o_gemm_ffma / b2o_gemv_ffma): the bit-exact yardstick of the product's FFMA GEMM / GEMV kernels ------
U32 = 2.0 ** -24


def gamma(n):
    return n * U32 / (1 - n * U32)


def test_gemm_ffma_known_answers():
    data = np.arange(1, 13, dtype=np.float32)
    A, B = data[:6], data
    At = np.array([1, 4, 2, 5, 3, 6], np.float32)
    Bt = np.array([1, 5, 9, 2, 6, 10, 3, 7, 11, 4, 8, 12], np.float32)
    want = np.array([38, 44, 50, 56, 83, 98, 113, 128], np.float32).reshape(2, 4)
    z = np.zeros((2, 4), np.float32)
    for tA, tB, a, b in ((0, 0, A, B), (1, 0, At, B), (1, 1, At, Bt), (0, 1, A, Bt)):
        out = o.gemm_ffma(tA, tB, 2, 4, 3, 1.0, a, b, 0.0, z)
        assert np.array_equal(out, np.broadcast_to(want, out.shape)), (tA, tB)
        # alpha and beta: 0.5 * AB + 2 * C0 is exact in every contraction
        c0 = np.arange(8, dtype=np.float32).reshape(2, 4)
        out = o.gemm_ffma(tA, tB, 2, 4, 3, 0.5, a, b, 2.0, c0)
        assert np.array_equal(out, np.broadcast_to(0.5 * want + 2 * c0, out.shape))
    # K = 0: beta * C exactly; alpha * (+0) keeps alpha's sign where beta = 0
    c0 = np.array([[1.5, -2.0]], np.float32)
    assert np.array_equal(o.gemm_ffma(0, 0, 1, 2, 0, 1.0, np.zeros(1, np.float32), np.zeros(1, np.float32), -2.0, c0)[0], -2 * c0)
    neg = o.gemm_ffma(0, 0, 1, 2, 0, -3.0, np.zeros(1, np.float32), np.zeros(1, np.float32), 0.0, c0)
    assert (neg.view(np.int32) == np.float32(-0.0).view(np.int32)).all()


def test_gemv_ffma_known_answers():
    A = np.arange(1, 7, dtype=np.float32)
    assert np.array_equal(o.gemv_ffma(0, 2, 3, 1.0, A, A[:3], 0.0, np.zeros(2, np.float32))[0], [14, 32])
    assert np.array_equal(o.gemv_ffma(1, 2, 3, 1.0, A, A[:2], 0.0, np.zeros(3, np.float32))[0], [9, 12, 15])
    assert np.array_equal(o.gemv_ffma(0, 3, 2, 1.0, A, A[:2], 0.0, np.zeros(3, np.float32))[0], [5, 11, 17])
    assert np.array_equal(o.gemv_ffma(1, 3, 2, 1.0, A, A[:3], 1.0, np.ones(2, np.float32))[2], [23, 29])


def test_gemm_ffma_padded_tail_turns_minus_zero_into_plus_zero():
    """sgemm_simt_kernel runs 16-wide K tiles with zeros past K: fmaf(0, 0, -0) = +0.  A product that underflows to -0 in the last
    real step survives when K % 16 == 0 and is lost to the padding otherwise"""
    for K, sign in ((16, -0.0), (15, 0.0), (1, 0.0)):
        a = np.zeros(K, np.float32)
        b = np.zeros(K, np.float32)
        a[K - 1], b[K - 1] = -1e-30, 1e-30
        got = o.gemm_ffma(0, 1, 1, 1, K, 1.0, a, b, 0.0, np.zeros((1, 1), np.float32))[0]
        assert got.view(np.int32)[0, 0] == np.float32(sign).view(np.int32), (K, got)


@pytest.mark.parametrize("tA,tB", [(0, 0), (0, 1), (1, 0), (1, 1)])
@pytest.mark.parametrize("alpha,beta", [(1.0, 0.0), (-3.0, 1.0), (0.5, -2.0)])
def test_gemm_ffma_within_classic_bound(rng, tA, tB, alpha, beta):
    """|ffma - exact| <= gamma_{Kp + 2} (|alpha| sum_k |a_k b_k| + |beta c|): one rounding per chain step, two in the store"""
    M, N, K = 37, 29, 100
    a = rng.standard_normal((K, M) if tA else (M, K)).astype(np.float32)
    b = rng.standard_normal((N, K) if tB else (K, N)).astype(np.float32)
    c0 = rng.standard_normal((M, N)).astype(np.float32)
    opA = (a.T if tA else a).astype(np.float64)
    opB = (b.T if tB else b).astype(np.float64)
    exact = alpha * (opA @ opB) + beta * c0
    mag = abs(alpha) * (np.abs(opA) @ np.abs(opB)) + abs(beta) * np.abs(c0)
    out = o.gemm_ffma(tA, tB, M, N, K, alpha, a, b, beta, c0)
    for r in out:
        assert (np.abs(r - exact) <= gamma(112 + 2) * mag).all()
    if beta == 0.0:                                    # nothing to contract: one answer
        assert np.array_equal(out[0], out[1]) and np.array_equal(out[0], out[2])
    elif alpha == -3.0:                                # fl(-3 acc) rounds: the contractions differ somewhere
        assert not np.array_equal(out[0], out[1])


@pytest.mark.parametrize("tA", [0, 1])
def test_gemv_ffma_within_classic_bound(rng, tA):
    M, N = 300, 1000
    A = rng.standard_normal((M, N)).astype(np.float32)
    x = rng.standard_normal(M if tA else N).astype(np.float32)
    y0 = rng.standard_normal(N if tA else M).astype(np.float32)
    opA = (A.T if tA else A).astype(np.float64)
    exact = 0.5 * (opA @ x) + y0
    mag = 0.5 * (np.abs(opA) @ np.abs(x)) + np.abs(y0)
    steps = M if tA else (N + 31) // 32 + 5            # the chain (and, NoTrans, the five butterfly adds)
    for r in o.gemv_ffma(tA, M, N, 0.5, A, x, 1.0, y0):
        assert (np.abs(r - exact) <= gamma(steps + 2) * mag).all()


def test_ffma_emulators_are_order_sensitive(rng):
    """reversing the k order changes the bits on random data: a kernel that summed in another order would fail a bit-exact check"""
    M, N, K = 64, 64, 100
    a = rng.standard_normal((M, K)).astype(np.float32)
    b = rng.standard_normal((K, N)).astype(np.float32)
    z = np.zeros((M, N), np.float32)
    fwd = o.gemm_ffma(0, 0, M, N, K, 1.0, a, b, 0.0, z)[0]
    rev = o.gemm_ffma(0, 0, M, N, K, 1.0, a[:, ::-1], b[::-1], 0.0, z)[0]
    assert np.mean(fwd.view(np.int32) != rev.view(np.int32)) > 0.5
    # the GEMV's lane-strided chains and butterfly are not a sequential sum either
    A = rng.standard_normal((200, 1000)).astype(np.float32)
    x = rng.standard_normal(1000).astype(np.float32)
    n = o.gemv_ffma(0, 200, 1000, 1.0, A, x, 0.0, np.zeros(200, np.float32))[0]
    seq = o.gemv_ffma(1, 1000, 200, 1.0, np.ascontiguousarray(A.T), x, 0.0, np.zeros(200, np.float32))[0]
    assert np.mean(n.view(np.int32) != seq.view(np.int32)) > 0.5
    assert np.mean(o.ffma_match(n, np.stack([seq] * 3))) < 0.5


# ---- im2col: reference source compiled verbatim (test_im2col_kernel.cu:102-212 shapes) ------------
# golden/im2col_ref_sha256.json: SHA-256 of what the reference's own im2col.cpp (2-D and N-D, compiled verbatim by
# tests/golden/make_golden.py) returns for these inputs; equal digests = bit-identical outputs.
IM2COL_SHAPES = [
    # (C,H,W,k,s,p,d)  first row is test_im2col_kernel.cu's 500x15x15, k3 s2 d3 p0
    (500, 15, 15, (3, 3), (2, 2), (0, 0), (3, 3)),
    (3, 6, 5, (3, 3), (2, 2), (0, 0), (1, 1)),
    (4, 9, 11, (3, 5), (2, 1), (1, 2), (1, 1)),
    (2, 12, 10, (3, 3), (1, 2), (2, 1), (2, 3)),
    (3, 20, 20, (7, 7), (2, 2), (3, 3), (1, 1)),
    (1, 5, 5, (3, 3), (1, 1), (3, 3), (1, 1)),
]


@pytest.mark.parametrize("shape", IM2COL_SHAPES)
def test_im2col_col2im_bit_exact_vs_reference_source(rng, shape):
    import hashlib
    import json
    Cc, H, W, k, s, p, d = shape
    want = json.load(open(os.path.join(GOLD, "im2col_ref_sha256.json")))[str(shape)]
    sha = lambda a: hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()
    im = rng.standard_normal((Cc, H, W)).astype(np.float32)
    col = o.im2col(im, k, s, p, d)
    assert sha(col) == want["col"]
    colr = rng.standard_normal(col.shape).astype(np.float32)
    back = o.col2im(colr, (Cc, H, W), k, s, p, d)
    assert sha(back) == want["back"]
    # N-D restatement against the reference N-D source and against the 2-D path (TestNDAgainst2D :606)
    coln = o.im2col_nd(im, k, s, p, d)
    assert sha(coln) == want["col_nd"] and np.array_equal(coln, col)
    backn = o.col2im_nd(colr, (Cc, H, W), k, s, p, d)
    assert sha(backn) == want["back_nd"]


def test_im2col_3d_nd(rng):
    # 3 spatial axes (TestSimple3DConvolution :352 uses the N-D path)
    im = rng.standard_normal((2, 5, 6, 4)).astype(np.float32)
    k, s, p, d = (3, 2, 3), (2, 1, 1), (1, 0, 1), (1, 2, 1)
    col = o.im2col_nd(im, k, s, p, d)
    # brute-force definition
    out = [(im.shape[1 + a] + 2 * p[a] - (d[a] * (k[a] - 1) + 1)) // s[a] + 1 for a in range(3)]
    want = np.zeros((2 * 18, *out), np.float32)
    for c in range(2):
        for a in range(3):
            for b in range(2):
                for e in range(3):
                    r = ((c * 3 + a) * 2 + b) * 3 + e
                    for x in range(out[0]):
                        for y in range(out[1]):
                            for z in range(out[2]):
                                i0, i1, i2 = x * s[0] - p[0] + a * d[0], y * s[1] - p[1] + b * d[1], z * s[2] - p[2] + e * d[2]
                                if 0 <= i0 < 5 and 0 <= i1 < 6 and 0 <= i2 < 4:
                                    want[r, x, y, z] = im[c, i0, i1, i2]
    assert np.array_equal(col, want)
    if o.ref() is not None:
        ref = np.empty_like(col)
        o.ref().ref_im2col_nd_cpu(im, 3, np.asarray(im.shape, np.int32), np.asarray(col.shape, np.int32),
                                  np.asarray(k, np.int32), np.asarray(p, np.int32), np.asarray(s, np.int32),
                                  np.asarray(d, np.int32), ref)
        assert np.array_equal(col, ref)


def test_im2col_layer_known_positions(rng):
    # test_im2col_layer.cpp:63-77: top-left 3x3 block of the first output location equals the image patch
    im = rng.standard_normal((3, 6, 5)).astype(np.float32)
    col = o.im2col(im, 3, 2, 0, 1)
    for c in range(3):
        for i in range(3):
            for j in range(3):
                assert col[(c * 3 + i) * 3 + j, 0, 0] == im[c, i, j]


# ---- forward: vs the independent direct definition (caffe_conv's role, tol 1e-4 :255) ------------
@pytest.mark.parametrize("name,case", ALL_CASES, ids=[c[0] for c in ALL_CASES])
def test_forward_matches_direct_definition(rng, name, case):
    prm = make(o, case)
    x, w, b, _ = tensors(rng, prm)
    y = o.conv_forward(prm, x, w, b)
    yd = o.conv_direct(prm, x, w, b)
    assert y.shape == prm.y_shape()
    assert np.abs(y - yd).max() <= 1e-4 * max(1.0, float(np.abs(yd).max()))


def test_sobel_known_answer(rng):
    # test_convolution_layer.cpp:511-604: 3x3 Sobel == (3x1 [1 2 1], stride (2,1)) then (1x3 [-1 0 1], stride (1,2))
    x = rng.standard_normal((2, 3, 6, 4)).astype(np.float32)
    w = np.tile(np.array([-1, 0, 1, -2, 0, 2, -1, 0, 1], np.float32), 3).reshape(1, 3, 3, 3)
    y = o.conv_forward(o.ConvParams.make(2, 3, 6, 4, 1, 3, 2, 0, 1, 1, False), x, w)
    w1 = np.tile(np.array([1, 2, 1], np.float32), 3).reshape(1, 3, 3, 1)
    t = o.conv_forward(o.ConvParams.make(2, 3, 6, 4, 1, (3, 1), (2, 1), 0, 1, 1, False), x, w1)
    w2 = np.array([-1, 0, 1], np.float32).reshape(1, 1, 1, 3)
    y2 = o.conv_forward(o.ConvParams.make(2, 1, t.shape[2], t.shape[3], 1, (1, 3), (1, 2), 0, 1, 1, False), t, w2)
    assert y.shape == y2.shape
    assert np.abs(y - y2).max() <= 1e-4


# ---- backward: finite differences like GradientChecker (step 1e-2, threshold 1e-3) --------------
@pytest.mark.parametrize("name,case", REF_TEST_CASES, ids=[c[0] for c in REF_TEST_CASES])
def test_backward_gradient_check(rng, name, case):
    prm = make(o, case)
    x, w, b, _ = tensors(rng, prm, scale_w=1.0)
    # objective = 0.5*||y||^2 -> dy = y   (test_gradient_check_util.hpp:71-172)
    y = o.conv_forward(prm, x, w, b, acc64=True)
    dw, db, dx = o.conv_backward(prm, x, w, y, acc64=True)

    def loss(xx, ww, bb):
        yy = o.conv_forward(prm, xx, ww, bb, acc64=True).astype(np.float64)
        return 0.5 * float((yy * yy).sum())

    step, thr = 1e-2, 1e-3
    for arr, grad, which in ((x, dx, 0), (w, dw, 1), (b, db, 2)):
        if arr is None:
            continue
        flat = arr.reshape(-1)
        for idx in rng.choice(flat.size, size=min(12, flat.size), replace=False):
            old = flat[idx]
            flat[idx] = old + step
            lp = loss(x, w, b)
            flat[idx] = old - step
            lm = loss(x, w, b)
            flat[idx] = old
            est = (lp - lm) / (2 * step)
            got = float(grad.reshape(-1)[idx])
            scale = max(abs(est), abs(got), 1.0)
            assert abs(est - got) <= thr * scale * 5, (which, idx, est, got)


def test_backward_accumulates_param_diffs_and_overwrites_bottom(rng):
    prm = o.ConvParams.make(2, 3, 6, 4, 4, 3, 2, 0, 1, 1, True)
    x, w, b, dy = tensors(rng, prm)
    dw0, db0, dx0 = o.conv_backward(prm, x, w, dy)
    dw1, db1, dx1 = o.conv_backward(prm, x, w, dy, dw=dw0, db=db0)
    assert np.allclose(dw1, 2 * dw0, rtol=1e-6, atol=1e-6) and np.allclose(db1, 2 * db0, rtol=1e-6, atol=1e-6)
    assert np.array_equal(dx0, dx1)


# ---- SGD / LR ---------------------------------------------------------------------------------
def test_sgd_update_closed_form(rng):
    # GradientBasedSolverTest closed form (test_gradient_based_solver.cpp:228-364): with momentum m, lr, decay wd:
    #   h' = m*h + lr*(g + wd*w);  w' = w - h'
    n = 1001
    g, w, h = (rng.standard_normal(n).astype(np.float32) for _ in range(3))
    for l2 in (True, False):
        for clear in (True, False):
            g2, w2, h2 = o.sgd_update(g, w, h, 0.9, 0.01, 0.0005, l2=l2, clear_grads=clear)
            reg = w if l2 else np.sign(w)
            hh = 0.9 * h.astype(np.float64) + 0.01 * (g.astype(np.float64) + 0.0005 * reg)
            assert np.allclose(h2, hh, rtol=1e-6, atol=1e-7)
            assert np.allclose(w2, w - hh, rtol=1e-6, atol=1e-6)
            assert np.array_equal(g2, np.zeros_like(g2)) if clear else np.array_equal(g2, h2)
    # iter_size accumulation normalisation and 1/solver_count folding
    g2, w2, h2 = o.sgd_update(g, w, h, 0.0, 1.0, 0.0, grad_scale=0.25, iter_size=2)
    assert np.allclose(h2, g * 0.125, rtol=1e-6)


def test_learning_rate_policies():
    assert o.learning_rate("fixed", 10, 0.1) == pytest.approx(0.1)
    assert o.learning_rate("step", 25, 0.1, gamma=0.5, stepsize=10) == pytest.approx(0.1 * 0.25)
    assert o.learning_rate("exp", 3, 0.1, gamma=0.9) == pytest.approx(0.1 * 0.9 ** 3, rel=1e-6)
    assert o.learning_rate("inv", 100, 0.01, gamma=1e-4, power=0.75) == pytest.approx(0.01 * (1 + 1e-4 * 100) ** -0.75, rel=1e-6)
    # resnet50 solver: poly, power 2
    assert o.learning_rate("poly", 1200000, 0.001, power=2.0, max_iter=2400000) == pytest.approx(0.001 * 0.25, rel=1e-6)
    assert o.learning_rate("multistep", 5, 0.1, gamma=0.1, current_step=2) == pytest.approx(0.001, rel=1e-5)
    assert o.learning_rate("fixed", 5, 0.1, rampup_interval=10, rampup_lr=0.0) == pytest.approx(0.05)


def test_allreduce_avg(rng):
    bufs = [rng.standard_normal(77).astype(np.float32) for _ in range(4)]
    out = o.allreduce_avg(bufs)
    want = (bufs[0] + bufs[1] + bufs[2] + bufs[3]) * np.float32(0.25)
    for b in out:
        assert np.allclose(b, want, rtol=1e-6, atol=1e-7)


# ---- golden fixtures produced from oracle/_ref (tests/golden/make_golden.py) -----------------------
def test_oracle_matches_golden_fixtures():
    path = os.path.join(GOLD, "conv_ref_golden.npz")
    assert os.path.exists(path), "golden fixture missing: run tests/golden/make_golden.py in the build container"
    z = np.load(path)
    names = sorted(set(k.split("/")[0] for k in z.files))
    assert len(names) >= 6
    for nm in names:
        c = {k: int(v) for k, v in zip(z[nm + "/keys"], z[nm + "/vals"])}
        prm = o.ConvParams(*[c[f] for f, _ in o.ConvParams._fields_])
        x, w, dy = z[nm + "/x"], z[nm + "/w"], z[nm + "/dy"]
        b = z[nm + "/b"] if prm.has_bias else None
        y = o.conv_forward(prm, x, w, b)
        dw, db, dx = o.conv_backward(prm, x, w, dy)
        # reference leg used OpenBLAS sgemm (different summation order): fp32 round-off tolerance
        assert rel_err(y, z[nm + "/y"]) < 2e-6, nm
        assert rel_err(dw, z[nm + "/dw"]) < 5e-6, nm
        assert rel_err(dx, z[nm + "/dx"]) < 2e-6, nm
        if prm.has_bias:
            assert rel_err(db, z[nm + "/db"]) < 5e-6, nm
        # im2col part of the fixture is bit-exact (pure copy)
        col = o.im2col(x[0], (prm.kh, prm.kw), (prm.sh, prm.sw), (prm.ph, prm.pw), (prm.dh, prm.dw))
        assert np.array_equal(col, z[nm + "/col0"]), nm


# ---- fused solver updates: fp32 contraction forms and the float64 restatement ------------------------------------------------
import itertools  # noqa: E402

import solver_oracle as so  # noqa: E402

F32 = np.float32


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.int32)


def test_solver_known_answers():
    """hand-computed steps on exact values, every delta clamp, and the Adam rate"""
    hp = dict(so.KERNEL_HP, momentum=0.5)
    # SGD: gr = 1*0.5 + 0.125*2 = 0.75, h = 0.5*0.5 + 0.25*0.75 = 0.4375, w = 2 - 0.4375
    g, w, h, _ = o.solver_fp32("SGD", 0, [1.0], [2.0], [0.5], None, hp, 0.25, 0.125, True, 0.5, False)
    assert (g[0], w[0], h[0]) == (0.4375, 1.5625, 0.4375)
    # Nesterov: h' = 0.4375 as above, u = 1.5*0.4375 - 0.5*0.5 = 0.40625
    g, w, h, _ = o.solver_fp32("Nesterov", 0, [1.0], [2.0], [0.5], None, hp, 0.25, 0.125, True, 0.5, False)
    assert (g[0], w[0], h[0]) == (0.40625, 1.59375, 0.4375)
    # L1: reg = sign(w) = -1, gr = 1 - 0.25 = 0.75
    g, w, h, _ = o.solver_fp32("SGD", 0, [1.0], [-2.0], [0.0], None, hp, 1.0, 0.25, False, 1.0, True)
    assert (g[0], w[0], h[0]) == (0.0, -2.75, 0.75)
    # the delta clamps: below the clamp the clamp, at it and above it delta itself
    for kind, clamp in (("AdaGrad", F32(1e-3)), ("RMSProp", F32(1e-4)), ("AdaDelta", F32(1e-3)), ("Adam", F32(1e-4))):
        for delta, used in ((1e-8, clamp), (float(clamp), clamp), (1e-2, F32(1e-2))):
            p = dict(hp, delta=delta, rms_decay=0.75, momentum=0.75, beta1=0.75, beta2=0.75)
            g, w, h, h2 = o.solver_fp32(kind, 0, [2.0], [1.0], [12.0], [5.0], p, 0.5, 0.0, True, 1.0, False)
            if kind == "AdaGrad":       # h = 12 + 4 = 16, u = 1 / (4 + d)
                want_h, want_u = 16.0, F32(1) / (F32(4) + used)
            elif kind == "RMSProp":     # h = 0.75*12 + 0.25*4 = 10, u = 1 / (sqrt(10) + d)
                want_h, want_u = 10.0, F32(1) / (np.sqrt(F32(10)) + used)
            elif kind == "AdaDelta":    # h = 10, gr = 2 sqrt((5 + d) / (10 + d)), h2 = 0.75*5 + 0.25 gr^2, u = gr / 2
                want_h = 10.0
                gr = F32(2) * np.sqrt((F32(5) + used) / (F32(10) + used))
                want_u = F32(0.5) * gr
                assert h2[0] == F32(3.75) + (F32(0.25) * gr) * gr
            else:                       # m = 0.75*12 + 0.25*2 = 9.5, v = 0.75*5 + 0.25*4 = 4.75, u = 0.5*9.5 / (sqrt(4.75) + d)
                want_h, want_u = 9.5, F32(4.75) / (np.sqrt(F32(4.75)) + used)
                assert h2[0] == 4.75
            assert h[0] == want_h and g[0] == want_u, (kind, delta)
            assert w[0] == F32(1) - want_u, (kind, delta)
    # Adam's first step from zero history with the bias-corrected rate lr*sqrt(1-b2)/(1-b1) moves w by lr*sign(g), less eps's
    # share: lr / (1 + eps / (sqrt(1-b2) |g|))
    b1, b2, lr = 0.9, 0.999, 0.01
    rate = float(F32(lr) * so.adam_correction(b1, b2, 1))
    gin = np.array([3.0, -0.5, 40.0], F32)
    g, w, h, h2 = o.solver_fp32("Adam", 0, gin, np.zeros(3), np.zeros(3), np.zeros(3), dict(hp, beta1=b1, beta2=b2), rate, 0.0,
                                True, 1.0, False)
    eps = 1e-4                                                  # delta 1e-8, clamped
    np.testing.assert_allclose(-w, lr * np.sign(gin) / (1 + eps / (np.sqrt(1 - b2) * np.abs(gin))), rtol=1e-5)


def test_solver_sign_of_zero():
    """w = +-0 under L1 regularises by +0 (sign(0) = 0), so an otherwise zero step keeps each zero's sign; a step of -0
    turns w = -0 into +0 (-0 - -0 = +0) -- in every form"""
    hp = dict(so.KERNEL_HP, momentum=0.5)
    w0 = np.array([0.0, -0.0, 0.0, -0.0], F32)
    for form in o.solver_forms("SGD"):
        g, w, h, _ = o.solver_fp32("SGD", form, np.zeros(4), w0, np.zeros(4), None, hp, 0.1, 0.01, False, 1.0, False)
        assert list(_bits(w)) == list(_bits(w0)) and list(_bits(g)) == [0] * 4
        # L1, decay 0: sign(-0) = +0 gives gr = -0 + +0 = +0, sign(-1) = -1 gives gr = -0 + -0 = -0
        g, w, h, _ = o.solver_fp32("SGD", form, [-0.0, -0.0], [-0.0, -1.0], [-0.0, -0.0], None, hp, 0.5, 0.0, False, 1.0, False)
        assert list(_bits(h)) == list(_bits(np.array([0.0, -0.0], F32))), form
        assert _bits(w)[1] == _bits(F32(-1.0)) and list(_bits(g)) == list(_bits(np.array([0.0, -0.0], F32)))
        # L2, decay 0, w = -0: gr = -0 + (-0)*0 = -0, h = -0, and w = -0 - (-0) = +0
        g, w, h, _ = o.solver_fp32("SGD", form, [-0.0], [-0.0], [-0.0], None, hp, 0.5, 0.0, True, 1.0, False)
        assert (_bits(h)[0], _bits(w)[0], _bits(g)[0]) == (_bits(F32(-0.0)), 0, _bits(F32(-0.0))), form


def test_solver_subnormals_are_kept():
    """fp32 subnormals are neither flushed on input nor on output: 3*2^-149 halved rounds to even (2*2^-149), a subnormal
    gradient steps w by itself"""
    tiny = F32(3 * 2.0 ** -149)
    g, w, h, _ = o.solver_fp32("SGD", 0, [0.0], [0.0], [tiny], None, dict(so.KERNEL_HP, momentum=0.5), 0.0, 0.0, True, 1.0, False)
    assert h[0] == F32(2 * 2.0 ** -149) and w[0] == -F32(2 * 2.0 ** -149)
    sub = F32(2.0 ** -140)
    g, w, h, _ = o.solver_fp32("SGD", 0, [sub], [0.0], [0.0], None, dict(so.KERNEL_HP, momentum=0.0), 1.0, 0.0, True, 1.0, False)
    assert w[0] == -sub and h[0] == sub


@pytest.mark.parametrize("kind", so.KINDS)
@pytest.mark.parametrize("l2", [True, False], ids=["L2", "L1"])
@pytest.mark.parametrize("clear", [True, False], ids=["clear", "keep"])
def test_solver_forms_within_float64_bound_and_distinct(kind, l2, clear):
    """every fp32 contraction form lies within the float64 restatement's derived bound on data over several binades with
    subnormals and +-0, at every delta regime; and on that data every pair of forms differs in some element, so that a kernel
    matching one form pins its contraction"""
    rng = np.random.default_rng(7)
    n = 20000
    g, w, h, h2 = so.wide_inputs(rng, n, kind)
    worst = 0.0
    for delta in (1e-8, 1e-3, 1e-2):
        hp = dict(so.KERNEL_HP, delta=delta, momentum=0.0 if kind in ("AdaGrad", "RMSProp") else 0.9)
        vals, bounds = o.solver_f64(kind, g, w, h, h2, hp, 0.3, 0.7, l2, 1 / 3, clear)
        outs = {}
        for form in o.solver_forms(kind):
            out = o.solver_fp32(kind, form, g, w, h, h2, hp, 0.3, 0.7, l2, 1 / 3, clear)
            for k in range(4):
                err = np.abs(out[k].astype(np.float64) - vals[k])
                assert np.all(err <= bounds[k] * (1 + 2.0 ** -20)), (kind, form, k, float(np.max(err / np.maximum(bounds[k], 1e-300))))
                worst = max(worst, float(np.max(err / np.maximum(bounds[k], 1e-300))))
            outs[form] = np.concatenate([_bits(a) for a in out])
        if delta == 1e-2:
            same = [(a, b) for a, b in itertools.combinations(outs, 2) if np.array_equal(outs[a], outs[b])]
            # L1: decay*sign(w) is exact, so fusing it changes nothing; clear: g is 0 in every form.  Nothing else may coincide.
            allowed = {(a, b) for a, b in same if not l2 and (a ^ b) in (2,)}
            assert set(same) == allowed, (kind, same[:4])
    print(f"[solver oracle] {kind} L2={l2} clear={clear}: worst |fp32 - f64| / bound = {worst:.3f}")


@pytest.mark.parametrize("kind", so.KINDS)
def test_solver_dyadic_data_makes_every_form_equal(kind):
    """on dyadic_inputs every product that meets a sum is exact, so every form equals the plain numpy fp32 restatement bit for
    bit -- AdaDelta's h2 and w excepted (they follow a rounded square root) -- which lets the GPU suite check such data against
    numpy whatever the compiler contracts"""
    rng = np.random.default_rng(11)
    g, w, h, h2 = so.dyadic_inputs(rng, 50000, kind)
    lrs, decays = so.dyadic_rates(rng, 6)
    for (lr, decay), l2, clear in itertools.product(zip(lrs, decays), (True, False), (True, False)):
        want = so.kernel_fp32(kind, g, w, h, h2, so.DYADIC_HP, lr, decay, l2, 0.125, clear)
        for form in o.solver_forms(kind):
            got = o.solver_fp32(kind, form, g, w, h, h2, so.DYADIC_HP, lr, decay, l2, 0.125, clear)
            for k in range(4):
                if kind == "AdaDelta" and k in (1, 3):
                    continue
                assert np.array_equal(_bits(got[k]), _bits(want[k])), (kind, form, k, lr, decay, l2, clear)

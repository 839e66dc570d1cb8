"""Per-element tests of the non-convolution kernels (csrc/layers.cu, csrc/layers_fused.cu, the bias kernels of csrc/conv_simt.cu)
against the float64 oracle (oracle/layers_oracle.py), at the shapes, routes and edges where they can go wrong.

The blob-level rel_err of test_layers_gpu.py divides the worst error by the largest value in the blob, so a small element that is
badly wrong goes unseen.  Here every element is judged on its own: by exact equality where the arithmetic allows it (comparisons,
copies, one rounding, integer data), else against a bound of the form c * 2^-24 * sum|terms| stated beside each op.

Every output is a Guarded buffer (tests/cases.py): NaN-prefilled, so an element never written shows up, with sentinel guard bands
that must be untouched.  Inputs sit in guarded buffers too, so a kernel that reads a little past its input stays inside memory
the test owns.  A second call must give the same bits.

Pooling picks one of five kernels from the shape and the alignment of y, mask and dx (include/b2c.h, b2c_pool_route).  Each
pooling case states the route and Ho x Wo it exists for and checks them through b2c_debug_pool_plan, with the pointers of the
real call, before it runs; shapes are chosen for 132 SMs (only the row kernel's grid depends on the SM count, not its route).
The same case then runs with y and mask, or dx, 4 bytes off alignment: that takes the scalar or row kernel, which must give the
same bits as the window or quad kernel.  The entry points read x and dy one float at a time, so only the outputs move."""
import ctypes as C

import numpy as np
import pytest

from oracle import layers_oracle as lo
from cases import Guarded

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import caffe_mpi_b200 as m  # noqa: E402
from caffe_mpi_b200 import capi  # noqa: E402

U = 2.0 ** -24                               # unit roundoff of float32
FLT_MIN = float(np.finfo(np.float32).tiny)


def st():
    return capi._stream()


def put(a, off=0):
    """a device copy of host array `a` (float32 or int32) inside a guarded buffer, `off` floats past a 16-byte boundary"""
    return Guarded(a.size, off, a)


def bits(a):
    return np.ascontiguousarray(a).view(np.int32)


def within(got, ref, bound, what):
    """|got - ref| <= bound, element by element; no NaN"""
    got64, ref64 = got.astype(np.float64), ref.astype(np.float64)
    assert not np.isnan(got64).any(), f"{what}: NaN (an element never written)"
    err = np.abs(got64 - ref64)
    bad = np.argwhere(err > bound)
    assert bad.size == 0, (f"{what}: {len(bad)} elements outside the bound, first at {tuple(bad[0])}: got {got64[tuple(bad[0])]!r}, "
                           f"want {ref64[tuple(bad[0])]!r}, bound {np.broadcast_to(bound, err.shape)[tuple(bad[0])]!r}")


def equal(got, ref, what):
    """the same values (the sign of a zero is not compared); no NaN"""
    assert not np.isnan(got.astype(np.float64)).any(), f"{what}: NaN (an element never written)"
    bad = np.argwhere(got != ref)
    assert bad.size == 0, (f"{what}: {len(bad)} elements differ, first at {tuple(bad[0])}: got {got[tuple(bad[0])]!r}, "
                           f"want {ref[tuple(bad[0])]!r}")


# ============================================================ pooling
# (id, NC, H, W, kernel, stride, pad, method, (Ho, Wo), forward route and Q, backward route and rows per block)
MAX, AVE = 0, 1
SQ = ((3, 3), (2, 2), (0, 0))        # the ResNet / GoogLeNet / AlexNet pool: 3x3 / stride 2 / no pad
IN = ((3, 3), (1, 1), (1, 1))        # the Inception branch pool: 3x3 / stride 1 / pad 1
POOL_CASES = [
    ("resnet_pool1_112", 512, 112, 112, *SQ, MAX, (56, 56), ("max_window", 4), ("max_bwd_quad", 0)),
    ("googlenet_56", 24, 56, 56, *SQ, MAX, (28, 28), ("max_window", 4), ("max_bwd_quad", 0)),
    ("googlenet_28", 24, 28, 28, *SQ, MAX, (14, 14), ("max_window", 2), ("max_bwd_quad", 0)),
    ("googlenet_14", 24, 14, 14, *SQ, MAX, (7, 7), ("max_scalar", 0), ("max_bwd_row", 9)),
    ("inception_28", 24, 28, 28, *IN, MAX, (28, 28), ("max_window", 4), ("max_bwd_quad", 0)),
    ("inception_14", 24, 14, 14, *IN, MAX, (14, 14), ("max_window", 2), ("max_bwd_row", 9)),
    ("inception_12", 10, 12, 12, *IN, MAX, (12, 12), ("max_window", 4), ("max_bwd_quad", 0)),
    ("inception_7", 24, 7, 7, *IN, MAX, (7, 7), ("max_scalar", 0), ("max_bwd_row", 18)),
    ("alexnet_55_grid_stride", 6144, 55, 55, *SQ, MAX, (27, 27), ("max_scalar", 0), ("max_bwd_row", 2)),
    ("alexnet_27", 24, 27, 27, *SQ, MAX, (13, 13), ("max_scalar", 0), ("max_bwd_row", 4)),
    ("alexnet_13", 24, 13, 13, *SQ, MAX, (6, 6), ("max_window", 2), ("max_bwd_row", 9)),
    ("vgg_224", 4, 224, 224, (2, 2), (2, 2), (0, 0), MAX, (112, 112), ("max_window", 4), ("max_bwd_quad", 0)),
    ("vgg_16", 10, 16, 16, (2, 2), (2, 2), (0, 0), MAX, (8, 8), ("max_window", 4), ("max_bwd_quad", 0)),
    ("vgg_14", 24, 14, 14, (2, 2), (2, 2), (0, 0), MAX, (7, 7), ("max_scalar", 0), ("max_bwd_row", 9)),
    ("rect_30x44", 12, 30, 44, *SQ, MAX, (15, 22), ("max_window", 2), ("max_bwd_quad", 0)),
    ("rect_44x30", 12, 44, 30, *SQ, MAX, (22, 15), ("max_scalar", 0), ("max_bwd_row", 4)),
    ("ceil_partial_last_window_10x16", 12, 10, 16, *SQ, MAX, (5, 8), ("max_window", 4), ("max_bwd_quad", 0)),
    ("padded_window_15", 12, 15, 15, (3, 3), (2, 2), (1, 1), MAX, (8, 8), ("max_window", 4), ("max_bwd_row", 8)),
    ("padded_8", 12, 8, 8, (3, 3), (2, 2), (1, 1), MAX, (5, 5), ("max_scalar", 0), ("max_bwd_quad", 0)),
    ("padded_9", 12, 9, 9, (3, 3), (2, 2), (1, 1), MAX, (5, 5), ("max_scalar", 0), ("max_bwd_row", 14)),
    ("padded_20", 10, 20, 20, (3, 3), (2, 2), (1, 1), MAX, (11, 11), ("max_scalar", 0), ("max_bwd_quad", 0)),
    ("wide_row_5x130", 12, 5, 130, *IN, MAX, (5, 130), ("max_window", 2), ("max_bwd_row", 1)),
    ("anisotropic_11x13", 12, 11, 13, (3, 2), (2, 1), (1, 0), MAX, (6, 12), ("max_scalar", 0), ("max_bwd_row", 9)),
    ("global_max_7", 12, 7, 7, (7, 7), (1, 1), (0, 0), MAX, (1, 1), ("max_scalar", 0), ("max_bwd_row", 18)),
    ("k1_s2_9", 12, 9, 9, (1, 1), (2, 2), (0, 0), MAX, (5, 5), ("max_scalar", 0), ("max_bwd_row", 14)),
    ("w3_6x3", 12, 6, 3, (2, 2), (2, 2), (0, 0), MAX, (3, 2), ("max_window", 2), ("max_bwd_row", 42)),
    ("w1_5x1_128_rows_per_block", 300, 5, 1, (1, 1), (1, 1), (0, 0), MAX, (5, 1), ("max_scalar", 0), ("max_bwd_row", 128)),
    ("ave_resnet_global_7", 24, 7, 7, (7, 7), (1, 1), (0, 0), AVE, (1, 1), ("ave", 0), ("ave", 0)),
    ("ave_googlenet_aux_14", 24, 14, 14, (5, 5), (3, 3), (0, 0), AVE, (4, 4), ("ave", 0), ("ave", 0)),
    ("ave_padded_8", 24, 8, 8, (3, 3), (2, 2), (1, 1), AVE, (5, 5), ("ave", 0), ("ave", 0)),
    ("ave_2x2_odd_9", 24, 9, 9, (2, 2), (2, 2), (0, 0), AVE, (5, 5), ("ave", 0), ("ave", 0)),
    ("ave_rect_10x14", 24, 10, 14, (3, 2), (2, 3), (1, 0), AVE, (6, 5), ("ave", 0), ("ave", 0)),
]


def pool_plan(c, d, out, mask=None):
    _, NC, H, W, k, s, p, method = c[:8]
    return capi.pool_plan(method, d, NC, H, W, k, s, p, out.ptr().value, mask.ptr().value if mask is not None else 0)


def check_route(c, d, out, mask, want_route, want_aux):
    q = pool_plan(c, d, out, mask)
    Ho, Wo = c[8]
    aux = q["q"] if d == 0 else q["rpb"]
    assert (q["route"], q["Ho"], q["Wo"], aux) == (want_route, Ho, Wo, want_aux), \
        f"{'forward' if d == 0 else 'backward'} no longer takes route {want_route} ({want_aux}) with Ho x Wo = {Ho} x {Wo}: {q}"
    if want_route == "max_window":                   # the pure query agrees with the real call's pointers
        assert q["q"] in (2, 4) and (out.ptr().value | mask.ptr().value) % (4 * q["q"]) == 0


def pool_fwd(c, x, off=0, route=None):
    """b2c_pool_forward with y (and mask) `off` floats off alignment; returns (y, mask)"""
    _, NC, H, W, k, s, p, method, (Ho, Wo) = c[:9]
    X = put(x)
    Y, M = Guarded(NC * Ho * Wo, off), (Guarded(NC * Ho * Wo, off) if method == MAX else None)
    if route:
        check_route(c, 0, Y, M, *route)
    capi.check(m.lib().b2c_pool_forward(method, NC, H, W, k[0], k[1], s[0], s[1], p[0], p[1], X.ptr(), Y.ptr(),
                                        M.ptr() if M else None, st()))
    shape = (1, NC, Ho, Wo)
    return Y.read().reshape(shape), (M.read(np.int32).reshape(shape) if M else None)


def pool_bwd(c, dy, mask, off=0, route=None):
    _, NC, H, W, k, s, p, method = c[:8]
    DY, MK = put(dy), (put(mask) if mask is not None else None)
    DX = Guarded(NC * H * W, off)
    if route:
        check_route(c, 1, DX, None, *route)
    capi.check(m.lib().b2c_pool_backward(method, NC, H, W, k[0], k[1], s[0], s[1], p[0], p[1], DY.ptr(),
                                         MK.ptr() if MK else None, DX.ptr(), st()))
    return DX.read().reshape(1, NC, H, W)


def fwd_twice_and_unaligned(c, x, fwd_route):
    """the forward on its route, a second time (same bits), and with y and mask 4 bytes off (scalar kernel, same bits)"""
    y, mask = pool_fwd(c, x, 0, fwd_route)
    y2, mask2 = pool_fwd(c, x)
    assert np.array_equal(bits(y), bits(y2)) and (mask is None or np.array_equal(mask, mask2)), "forward: not bit-identical run to run"
    un_route = fwd_route if fwd_route[0] != "max_window" else ("max_scalar", 0)
    yu, masku = pool_fwd(c, x, 1, un_route)
    assert np.array_equal(bits(y), bits(yu)), f"forward: {un_route[0]} (y 4 bytes off) and {fwd_route[0]} give different bits"
    assert mask is None or np.array_equal(mask, masku), f"forward: {un_route[0]} and {fwd_route[0]} give different masks"
    return y, mask


def bwd_twice_and_unaligned(c, dy, mask, bwd_route):
    dx = pool_bwd(c, dy, mask, 0, bwd_route)
    assert np.array_equal(bits(dx), bits(pool_bwd(c, dy, mask))), "backward: not bit-identical run to run"
    H, W = c[2], c[3]
    un_route = bwd_route if bwd_route[0] != "max_bwd_quad" else ("max_bwd_row", 1 if W >= 128 else 128 // W)
    dxu = pool_bwd(c, dy, mask, 1, un_route)
    assert np.array_equal(bits(dx), bits(dxu)), f"backward: {un_route[0]} (dx 4 bytes off) and {bwd_route[0]} give different bits"
    return dx


@pytest.mark.parametrize("c", POOL_CASES, ids=[c[0] for c in POOL_CASES])
def test_pooling(rng, c):
    _, NC, H, W, k, s, p, method, (Ho, Wo), fwd_route, bwd_route = c
    assert (lo.pooled_extent(H, k[0], s[0], p[0]), lo.pooled_extent(W, k[1], s[1], p[1])) == (Ho, Wo)
    shape = (1, NC, H, W)
    ntaps = k[0] * k[1]                     # the most terms any element of y or dx sums (windows overlapping one input <= taps)
    normal = rng.standard_normal(shape).astype(np.float32)
    if method == MAX:
        ties = np.maximum(np.round(2 * normal), 0).astype(np.float32)       # relu(round(2x)): zeros and small integers tie often
        for name, x in (("normal", normal), ("tie-heavy", ties)):
            # y and the first-maximum mask are selections: bit-exact
            y_ref, mask_ref = lo.pool_forward(x, MAX, k, s, p)
            y, mask = fwd_twice_and_unaligned(c, x, fwd_route)
            assert np.array_equal(bits(y), bits(y_ref)), f"{name} x: y differs from the oracle"
            bad = np.argwhere(mask != mask_ref)
            assert bad.size == 0, f"{name} x: mask differs at {len(bad)} outputs, first {tuple(bad[0])}: {mask[tuple(bad[0])]} vs {mask_ref[tuple(bad[0])]}"
            # dx with small-integer dy: sums of integers are exact in any order
            dyi = rng.integers(-8, 9, y.shape).astype(np.float32)
            equal(bwd_twice_and_unaligned(c, dyi, mask, bwd_route), lo.pool_backward(dyi, mask_ref, shape, MAX, k, s, p),
                  f"{name} x, integer dy: dx")
            # dx with normal dy: at most ntaps terms, any order: |err| <= ntaps * u * sum|dy terms| (the oracle's rounding included)
            dy = rng.standard_normal(y.shape).astype(np.float32)
            ref = lo.pool_backward(dy, mask_ref, shape, MAX, k, s, p)
            mag = lo.pool_backward(np.abs(dy), mask_ref, shape, MAX, k, s, p).astype(np.float64)
            within(pool_bwd(c, dy, mask), ref, ntaps * U * mag, f"{name} x, normal dy: dx")
        return
    if k == (2, 2) and s == (2, 2):
        # integer x and dy; every divisor (4, 2 or 1 where the last window is clipped) is a power of two: exact
        xi = rng.integers(-8, 9, shape).astype(np.float32)
        y_ref, _ = lo.pool_forward(xi, AVE, k, s, p)
        y, _ = fwd_twice_and_unaligned(c, xi, fwd_route)
        equal(y, y_ref, "integer x: AVE y")
        dyi = rng.integers(-8, 9, y.shape).astype(np.float32)
        equal(bwd_twice_and_unaligned(c, dyi, None, bwd_route), lo.pool_backward(dyi, None, shape, AVE, k, s, p), "integer dy: AVE dx")
    # y = (sum of <= ntaps floats) / padded window size: |err| <= (ntaps + 1) * u * sum|x| / size
    x = normal
    y_ref, _ = lo.pool_forward(x, AVE, k, s, p)
    mag = lo.pool_forward(np.abs(x), AVE, k, s, p)[0].astype(np.float64)
    y, _ = fwd_twice_and_unaligned(c, x, fwd_route)
    within(y, y_ref, (ntaps + 1) * U * mag, "AVE y")
    # dx = sum over <= ntaps windows of dy / size, each quotient rounded: |err| <= (ntaps + 1) * u * sum|dy / size|
    dy = rng.standard_normal(y.shape).astype(np.float32)
    ref = lo.pool_backward(dy, None, shape, AVE, k, s, p)
    mag = lo.pool_backward(np.abs(dy), None, shape, AVE, k, s, p).astype(np.float64)
    within(bwd_twice_and_unaligned(c, dy, None, bwd_route), ref, (ntaps + 1) * U * mag, "AVE dx")


# ============================================================ elementwise: ReLU, Eltwise SUM, their fused forms
SIZES = [1, 3, 4, 5, 4097, 2 ** 20 + 3]


def _relu_fwd(L, n, ins, outs, slope):
    return L.b2c_relu_forward(n, ins[0], outs[0], C.c_float(slope), st())


def _relu_bwd(L, n, ins, outs, slope):
    return L.b2c_relu_backward(n, ins[0], ins[1], outs[0], C.c_float(slope), st())


def _add(L, n, ins, outs, slope):
    return L.b2c_add(n, ins[0], ins[1], outs[0], st())


def _add_relu(L, n, ins, outs, slope):
    return L.b2c_add_relu(n, ins[0], ins[1], outs[0], st())


def _relu_bwd2(which):
    def call(L, n, ins, outs, slope):
        a = outs[0] if which in ("both", "a") else None
        b = outs[-1] if which in ("both", "b") else None
        return L.b2c_relu_backward2(n, ins[0], ins[1], a, b, st())
    return call


def _oracle(op, ins, slope):
    f = np.float32(slope)
    if op.startswith("relu_forward"):
        return lo.relu_forward(ins[0], f)
    if op.startswith("relu_backward_"):
        return lo.relu_backward(ins[0], ins[1], f)
    if op == "add":
        return ins[0] + ins[1]
    if op == "add_relu":
        return lo.relu_forward(ins[0] + ins[1])
    return lo.relu_backward(ins[0], ins[1])                                # relu_backward2: dy * (y > 0)


# (name, call, inputs, outputs, slope)
EW_OPS = [
    ("relu_forward_slope0", _relu_fwd, 1, 1, 0.0),
    ("relu_forward_slope0.1", _relu_fwd, 1, 1, 0.1),
    ("relu_backward_slope0", _relu_bwd, 2, 1, 0.0),
    ("relu_backward_slope0.1", _relu_bwd, 2, 1, 0.1),
    ("add", _add, 2, 1, 0.0),
    ("add_relu", _add_relu, 2, 1, 0.0),
    ("relu_backward2_both", _relu_bwd2("both"), 2, 2, 0.0),
    ("relu_backward2_dx_b_null", _relu_bwd2("a"), 2, 1, 0.0),
    ("relu_backward2_dx_a_null", _relu_bwd2("b"), 2, 1, 0.0),
]


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("op", EW_OPS, ids=[o[0] for o in EW_OPS])
def test_elementwise(rng, op, n):
    """one comparison, one product or one sum per element: exactly the numpy oracle's float32 value, with every pointer 16-byte
    aligned (float4 passes) and with every pointer 4 bytes off (one float at a time); the two give the same bits"""
    name, call, nin, nout, slope = op
    L = m.lib()
    ins = [rng.standard_normal(n).astype(np.float32) for _ in range(nin)]
    if nin == 2 and name.startswith("relu_backward"):
        ins[1][::7] = 0.0                                                   # x (or y) exactly 0 takes the slope / mask side
    want = _oracle(name, ins, slope).astype(np.float32)
    assert want.dtype == np.float32
    runs = []
    for off in (0, 1):
        I = [put(a, off) for a in ins]
        O = [Guarded(n, off) for _ in range(nout)]
        capi.check(call(L, n, [t.ptr() for t in I], [t.ptr() for t in O], slope))
        for t in O:
            got = t.read()
            equal(got, want, f"{name}, n = {n}, {'4 bytes off' if off else 'aligned'}")
            runs.append(got)
    for a in runs[1:]:
        assert np.array_equal(bits(a), bits(runs[0])), f"{name}, n = {n}: outputs or alignments give different bits"


IN_PLACE = [("relu_forward_y_is_x", 0.0), ("relu_forward_y_is_x_slope0.1", 0.1), ("add_y_is_a", 0.0), ("add_relu_y_is_a", 0.0)]


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("op,slope", IN_PLACE, ids=[o[0] for o in IN_PLACE])
def test_elementwise_in_place(rng, op, slope, n):
    """y == x (the prototxt's in-place ReLU) and y == a (Eltwise into its first bottom), aligned and 4 bytes off"""
    L = m.lib()
    a, b = rng.standard_normal(n).astype(np.float32), rng.standard_normal(n).astype(np.float32)
    if op.startswith("relu"):
        want = lo.relu_forward(a, np.float32(slope))
    else:
        want = a + b if op == "add_y_is_a" else lo.relu_forward(a + b)
    for off in (0, 1):
        A, B = Guarded(n, off, a), put(b, off)
        if op.startswith("relu"):
            rc = L.b2c_relu_forward(n, A.ptr(), A.ptr(), C.c_float(slope), st())
        elif op == "add_y_is_a":
            rc = L.b2c_add(n, A.ptr(), B.ptr(), A.ptr(), st())
        else:
            rc = L.b2c_add_relu(n, A.ptr(), B.ptr(), A.ptr(), st())
        capi.check(rc)
        equal(A.read(), want.astype(np.float32), f"{op}, n = {n}, {'4 bytes off' if off else 'aligned'}")


# ============================================================ transpose
@pytest.mark.parametrize("rows,cols", [(1, 1), (1, 5000), (5000, 1), (31, 33), (32, 32), (33, 31), (64, 1000), (1000, 4097)])
def test_transpose(rng, rows, cols):
    """dst[c][r] = src[r][c]: a copy, bit-exact, every element written, nothing outside dst"""
    src = rng.standard_normal((rows, cols)).astype(np.float32)
    S, D = put(src), Guarded(rows * cols)
    capi.check(m.lib().b2c_transpose(rows, cols, S.ptr(), D.ptr(), st()))
    got = D.read().reshape(cols, rows)
    assert np.array_equal(bits(got), bits(np.ascontiguousarray(src.T)))


def test_transpose_refusals():
    """src == dst and more than 65535 * 32 rows (the grid's y limit) are refused before any launch"""
    L = m.lib()
    S, D = Guarded(64), Guarded(64)
    assert L.b2c_transpose(8, 8, S.ptr(), S.ptr(), st()) == -1
    assert L.b2c_transpose(65535 * 32 + 1, 1, S.ptr(), D.ptr(), st()) == -1
    assert np.isnan(D.read()).all()                                         # untouched: still NaN inside, sentinels outside


# ============================================================ bias
@pytest.mark.parametrize("P", [1, 49, 3136])
def test_bias_forward(rng, P):
    """y[n][o][p] += bias[o]: one rounding, exactly the float32 sum"""
    N, O = 3, 7
    y0 = rng.standard_normal((N, O, P)).astype(np.float32)
    b = rng.standard_normal(O).astype(np.float32)
    Y, B = Guarded(y0.size, 0, y0), put(b)
    capi.check(m.lib().b2c_bias_forward(N, O, P, B.ptr(), Y.ptr(), st()))
    equal(Y.read().reshape(N, O, P), y0 + b[None, :, None], "bias forward")


BIAS_SHAPES = {1: (1, 1), 3: (1, 3), 4: (2, 2), 49: (7, 7), 3136: (56, 56)}


def _bias_grad(api, N, O, P, dy, db0, off):
    DY, DB = put(dy, off), Guarded(O, 0, db0)
    if api == "ip":
        capi.check(m.lib().b2c_bias_backward(N, O, P, DY.ptr(), DB.ptr(), st()))
    else:
        H, W = BIAS_SHAPES[P]
        d = m.ConvDesc(capi.ConvParams.make(N, 1, H, W, O, 1, 1, 0, 1, 1, True))
        capi.check(m.lib().b2c_conv_backward_bias(d._h, DY.ptr(), DB.ptr(), st()))
    return DB.read()


@pytest.mark.parametrize("N", [1, 37, 256])
@pytest.mark.parametrize("P", [1, 3, 4, 49, 3136])
@pytest.mark.parametrize("api", ["ip", "conv"])
def test_bias_backward(rng, api, P, N):
    """db[o] = db0[o] + sum_{n,p} dy[n][o][p] through b2c_bias_backward (InnerProduct, any P) and b2c_conv_backward_bias.
    One block per channel: each thread sums at most N * ceil(P / 256) values in order (a float4 first reduces its four in two
    levels), then a 5-level shuffle tree, an in-order sum over the 8 warps and the add onto db0, so no term passes through more
    than N * ceil(P / 256) + 16 roundings: |err| <= (N * ceil(P / 256) + 17) * u * (|db0| + sum|dy|), the oracle's own rounding
    included.  P = 1 leaves the
    whole sum to one thread.  With integer dy the sum is exact and db0 + it is one rounding: equal to the oracle."""
    O = 3
    c = N * -(-P // 256) + 17
    dy = rng.standard_normal((N, O, P)).astype(np.float32)
    db0 = rng.standard_normal(O).astype(np.float32)
    want = lo.bias_backward(dy, db0)
    mag = np.abs(db0).astype(np.float64) + np.abs(dy).astype(np.float64).sum(axis=(0, 2))
    got = _bias_grad(api, N, O, P, dy, db0, 0)
    within(got, want, c * U * mag, f"db, dy aligned (P % 4 == 0: float4 loads)")
    assert np.array_equal(bits(got), bits(_bias_grad(api, N, O, P, dy, db0, 0))), "db: not bit-identical run to run"
    un = _bias_grad(api, N, O, P, dy, db0, 1)                           # dy 4 bytes off: the scalar loads
    within(un, want, c * U * mag, "db, dy 4 bytes off")
    if P % 4:
        assert np.array_equal(bits(un), bits(got)), "db: dy 4 bytes off does not give the bits of the aligned scalar path"
    dyi = rng.integers(-8, 9, (N, O, P)).astype(np.float32)
    for off in (0, 1):
        equal(_bias_grad(api, N, O, P, dyi, db0, off), lo.bias_backward(dyi, db0), f"db, integer dy, offset {off}")


# ============================================================ softmax with loss
def _softmax(N, Cc, z, lab, loss_weight):
    L = m.lib()
    Z, LB = put(z), put(lab)
    P, LOSS, DX = Guarded(N * Cc), Guarded(1), Guarded(N * Cc)
    capi.check(L.b2c_softmax_loss_forward(N, Cc, Z.ptr(), LB.ptr(), P.ptr(), LOSS.ptr(), st()))
    prob = P.read().reshape(N, Cc)
    Pd = put(prob)
    capi.check(L.b2c_softmax_loss_backward(N, Cc, Pd.ptr(), LB.ptr(), C.c_float(loss_weight), DX.ptr(), st()))
    return prob, float(LOSS.read()[0]), DX.read().reshape(N, Cc)


@pytest.mark.parametrize("loss_weight", [1.0, 0.3])
@pytest.mark.parametrize("N,Cc", [(1, 1), (3, 10), (5, 31), (64, 1000), (257, 1000), (1000, 10), (2, 4097), (2, 21841)])
def test_softmax_loss(rng, N, Cc, loss_weight):
    """Logits x30 + 1000: the max subtraction is what keeps expf finite (z - max is exact: Sterbenz).  Labels 0 and C-1; the last
    row's label logit sits 200 below the row's minimum, so p[label] underflows and the term is clamped at -log(FLT_MIN).
    prob: expf (2 ulp), a sum of positive terms of depth ceil(C/256) + 10, 1/s, one product, the oracle's rounding:
      |err| <= c_p * u * p + FLT_MIN, c_p = ceil(C/256) + 16 (FLT_MIN: below the normal range there is no relative accuracy).
    loss: each term -logf(max(p, FLT_MIN)) is off by <= c_p * u (from p) + 2 u |term| (logf), the terms are summed with depth
      ceil(N/256) + 10 and scaled by 1/N (two roundings):  |err| <= c_p * u + (ceil(N/256) + 12) * u * mean|term| + 2 u |loss|.
    dx = (p - onehot) * (loss_weight / N) from the kernel's own prob: p - onehot, loss_weight in float32, the scale, the product and
      the oracle round once each:  |err| <= (c_p * u * p + FLT_MIN + 5 u |p - onehot|) * loss_weight / N."""
    z = (rng.standard_normal((N, Cc)) * 30 + 1000).astype(np.float32)
    lab = rng.integers(0, Cc, N).astype(np.float32)
    lab[0] = 0
    if N > 1:
        lab[1] = Cc - 1
    if Cc > 1:
        z[N - 1, int(lab[N - 1])] = z[N - 1].min() - 200
    prob, loss, dx = _softmax(N, Cc, z, lab, loss_weight)
    p_ref, loss_ref = lo.softmax_loss_forward(z, lab)
    if Cc == 1:                                                              # prob == 1, loss == dx == 0, exactly
        assert (prob == 1).all() and loss == 0 and (dx == 0).all(), (prob, loss, dx)
        return
    cp = -(-Cc // 256) + 16
    p64 = p_ref.astype(np.float64)
    within(prob, p_ref, cp * U * p64 + FLT_MIN, "prob")
    assert prob[N - 1, int(lab[N - 1])] < FLT_MIN, "the clamped row's p[label] did not underflow"
    terms = -np.log(np.maximum(p64[np.arange(N), lab.astype(np.int64)], FLT_MIN))
    lb = cp * U + (-(-N // 256) + 12) * U * terms.mean() + 2 * U * abs(float(loss_ref))
    assert abs(loss - float(loss_ref)) <= lb, (loss, float(loss_ref), lb)
    onehot = np.zeros_like(p64)
    onehot[np.arange(N), lab.astype(np.int64)] = 1
    dx_ref = lo.softmax_loss_backward(p_ref, lab, loss_weight)
    within(dx, dx_ref, (cp * U * p64 + FLT_MIN + 5 * U * np.abs(p64 - onehot)) * loss_weight / N, "dx")


# ============================================================ accuracy
@pytest.mark.parametrize("N", [1, 9, 1000])
@pytest.mark.parametrize("Cc", [1, 10, 33, 1000])
def test_accuracy(rng, N, Cc):
    """hits / N, exactly lo.accuracy: integer scores in [0, 4) tie often (equal scores rank the higher class first), every third
    row ties throughout, and labels -1 and C (the reference DCHECKs the range) count as misses.  N = 1000: 32 blocks of 8 warps."""
    L = m.lib()
    L.b2c_accuracy.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    z = rng.integers(0, 4, (N, Cc)).astype(np.float32)
    z[::3] = 1.5
    lab = rng.integers(0, Cc, N).astype(np.float32)
    lab[1::5] = -1
    lab[2::5] = Cc
    Z, LB = put(z), put(lab)
    for k in sorted({1, 5, Cc} & set(range(1, Cc + 1))):
        ACC, SCR = Guarded(1), torch.zeros(4, dtype=torch.uint8, device="cuda")
        capi.check(L.b2c_accuracy(N, Cc, k, Z.ptr().value, LB.ptr().value, ACC.ptr().value, SCR.data_ptr(), capi._stream().value))
        got, want = ACC.read()[0], lo.accuracy(z, lab, k)
        assert bits(np.float32(got)) == bits(np.float32(want)), (k, got, want)


# ============================================================ LRN across channels
# (id, shape, size, alpha, beta, k, spike)
LRN_CASES = [
    ("alexnet_rsqrt", (4, 96, 27, 27), 5, 1e-4, 0.75, 1.0, False),
    ("beta_0.5_powf", (2, 32, 7, 9), 5, 1e-4, 0.5, 2.0, False),
    ("size_1", (2, 8, 5, 5), 1, 1e-2, 0.75, 1.0, False),
    ("size_15_c3", (2, 3, 6, 6), 15, 1e-2, 0.75, 1.0, False),
    ("c1", (3, 1, 4, 4), 5, 1e-2, 0.75, 1.0, False),
    ("s1", (5, 20, 1, 1), 5, 1e-2, 0.75, 1.0, False),
    ("spike_alpha1", (2, 16, 6, 6), 5, 1.0, 0.75, 1.0, True),
]


def _window_sums(v, size, pre):
    """sum of v over channel window [c - pre, c - pre + size) clipped to [0, C), per (n, c, pixel), float64"""
    Cc = v.shape[1]
    out = np.empty_like(v)
    for c in range(Cc):
        out[:, c] = v[:, max(c - pre, 0):min(c - pre + size, Cc)].sum(axis=1)
    return out


@pytest.mark.parametrize("case", LRN_CASES, ids=[c[0] for c in LRN_CASES])
def test_lrn(rng, case):
    """The kernels keep the reference's running window sum over channels (lrn_layer.cpp; and its own lrn_layer.cu): channel c's
    sum is channel c-1's plus the head of the window minus its tail.  Each step rounds the two squares (or ratios) and the two
    updates, each by at most u times the window sums around it, so the sum at channel c carries an error of at most
      E(c) = 16 u * sum_{j <= c} Wabs(j),  Wabs = the window sum of x^2 (of |ratio| in backward).
    It grows along the channels and depends on the magnitudes that have passed through the window, not on the current one:
    with alpha = 1 and a channel of 1000s it is the reference algorithm's own error, not a kernel fault.  From it:
      scale: |err| <= alpha/size * E(c) + 3 u * scale           (alpha/size, the update and the oracle round once each)
      y = x * scale^-beta: |err| <= |y| * (beta * scale_bound / scale + 8 u)     (rsqrtf 2 ulp or powf 4 ulp, two products)
      dx = dy * scale^-beta - cr * x * sum(ratio), cr = 2 alpha beta / size (three roundings), ratio = dy * y / scale (two):
           |err| <= 8 u |dy scale^-beta| + cr |x| (E(c) + 8 u Rabs(c)) + 2 u |dx|,   Rabs = the window sum of |ratio|.
    The backward is fed the oracle's y and scale, so only its own roundings count."""
    _, shape, size, alpha, beta, k, spike = case
    N, Cc, H, W = shape
    S = H * W
    x = rng.standard_normal(shape).astype(np.float32)
    if spike:
        x *= np.float32(0.1)
        x[:, Cc // 2] = 1000.0
    dy = rng.standard_normal(shape).astype(np.float32)
    y_ref, s_ref = lo.lrn_forward(x, size, alpha, beta, k)
    dx_ref = lo.lrn_backward(x, y_ref, s_ref, dy, size, alpha, beta)
    L = m.lib()
    X = put(x)
    SC, Y = Guarded(x.size), Guarded(x.size)
    capi.check(L.b2c_lrn_forward(N, Cc, S, size, C.c_float(alpha), C.c_float(beta), C.c_float(k), X.ptr(), SC.ptr(), Y.ptr(), st()))
    scale, y = SC.read().reshape(shape), Y.read().reshape(shape)
    pre = (size - 1) // 2
    x64 = x.astype(np.float64)
    E = 16 * U * np.cumsum(_window_sums(x64 ** 2, size, pre), axis=1)
    s64 = s_ref.astype(np.float64)
    sb = alpha / size * E + 3 * U * s64
    within(scale, s_ref, sb, "scale")
    within(y, y_ref, np.abs(y_ref.astype(np.float64)) * (beta * sb / s64 + 8 * U), "y")
    DY, YR, SR, DX = put(dy), put(y_ref), put(s_ref), Guarded(x.size)
    capi.check(L.b2c_lrn_backward(N, Cc, S, size, C.c_float(alpha), C.c_float(beta), X.ptr(), YR.ptr(), SR.ptr(), DY.ptr(), DX.ptr(), st()))
    dx = DX.read().reshape(shape)
    ratio = np.abs(dy.astype(np.float64) * y_ref / s64)
    ipp = size - (size + 1) // 2
    Rabs = _window_sums(ratio, size, ipp)
    cr = 2.0 * alpha * beta / size
    bound = 8 * U * np.abs(dy) * s64 ** -beta + cr * np.abs(x64) * (16 * U * np.cumsum(Rabs, axis=1) + 8 * U * Rabs) \
        + 2 * U * np.abs(dx_ref.astype(np.float64))
    within(dx, dx_ref, bound, "dx")
    again = Guarded(x.size)
    capi.check(L.b2c_lrn_backward(N, Cc, S, size, C.c_float(alpha), C.c_float(beta), X.ptr(), YR.ptr(), SR.ptr(), DY.ptr(), again.ptr(), st()))
    assert np.array_equal(bits(again.read().reshape(shape)), bits(dx)), "dx: not bit-identical run to run"

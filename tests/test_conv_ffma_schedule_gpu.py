"""The exact-fp32 convolution paths, element by element: the FFMA direct kernels, the CAFFE engine and the host layer's N-D path.

All three are deterministic fp32 in a fixed order, so each is restated and held to its restatement bit for bit (int32 views: the
sign of a zero counts).  The blob-level max|err| / max|ref| of the older suites cannot see a small element that is badly wrong;
these checks can.

  * FFMA kernels (conv_simt.cu; b2c_conv_route / b2c_wgrad_route "simt"): oracle.conv_fwd_ffma / conv_dgrad_ffma /
    conv_wgrad_ffma restate their fmaf chains (the weight gradient's 256 lane-strided chains, warp butterflies and 8 ordered warp
    partials included).  They run every strided k > 1 data gradient (the four strided Inception-v2 layers on every training
    step), forward and data-gradient shapes past the gather table, and everything under ALGO_SIMT.  These kernels have no vector
    path: x, y, dy and dx 4 bytes off alignment must give the same bits.  Each case is also held to float64 within the bound
    derived in tests/test_conv_ffma_cpu.py, a second opinion should the restatement itself be wrong.
  * CAFFE engine (api.cu): per image im2col, per group b2c_sgemm, then the bias kernel (forward); sgemm TN then col2im (data
    gradient); per image sgemm NT with beta = 1 (weight gradient).  Restated with oracle.im2col / col2im / gemm_ffma.  Every GEMM
    the call issues is asserted on capi.sgemm_plan with the call's own pointers: the global defaults pick those routes, not the
    descriptor's math or algo.  A weight gradient whose per-image GEMMs run on the FFMA kernel is checked bit for bit with N = 1
    (one GEMM per group: one of the three admissible contractions of alpha * acc + beta * c), and with N > 1 exactly on integer
    data and under the float64 bound; one on the tensor cores exactly on integer data and under the GEMM suite's per-element
    bound summed over the images.
  * N-D path (ConvolutionLayer in host/b2caffe.cpp, 3-D convolutions and force_nd_im2col): per image im2col_nd + sgemm + the bias
    as a K = 1 GEMM against a ones row; backward sgemv for db, sgemm NT beta = 1 for dW, sgemm TN + col2im_nd for dx.  The layer's
    buffers come from cudaMalloc (256-byte aligned), so its GEMM plans are asserted at a 256-byte aligned base plus the call's
    offsets.  Param diffs accumulate over two Backward calls from a random start; dx is overwritten.

Harness: every output is a cases.Guarded buffer (NaN inside, sentinels around); the workspace is exactly b2c_conv_workspace_bytes
(a null pointer when that is 0) filled with 0xFF; dW starts at a random dw0; a second call gives the same bits."""
import ctypes as C

import numpy as np
import pytest

import oracle as o
from cases import Guarded, rel_err

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import caffe_mpi_b200 as m  # noqa: E402
from caffe_mpi_b200 import capi, host_api as h  # noqa: E402

U = 2.0 ** -24
SLACK = 1.0 + 2.0 ** -20
OPS = {"fwd": capi.OP_FORWARD, "dgrad": capi.OP_BACKWARD_DATA, "wgrad": capi.OP_BACKWARD_FILTER}


def gamma(n):
    return n * U / (1 - n * U)


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.int32)


def assert_bits(got, want, what):
    bad = np.argwhere(bits(got) != bits(want))
    assert bad.size == 0, (f"{what}: {len(bad)} of {got.size} elements differ in their bits, first at {tuple(bad[0])}: "
                           f"got {got[tuple(bad[0])]!r}, want {want[tuple(bad[0])]!r}")


def conv(N, C, H, W, O, k, s=1, p=0, d=1, G=1, bias=True):
    return dict(N=N, C=C, H=H, W=W, O=O, k=k, s=s, p=p, d=d, G=G, bias=bias)


def params(mod, c, **over):
    c = dict(c, **over)
    return mod.ConvParams.make(c["N"], c["C"], c["H"], c["W"], c["O"], c["k"], c["s"], c["p"], c["d"], c["G"], c["bias"])


def dptr(t):
    return t.data_ptr() if t is not None else 0


def vp(a):
    return C.c_void_p(a or None)


class Caller:
    """b2c_conv_forward / backward_data / backward_filter through the C ABI on host arrays: inputs `off` floats past a 256-byte
    boundary, the output a Guarded buffer as far off, the workspace exactly b2c_conv_workspace_bytes of 0xFF (null when 0).
    Keeps the device pointers of the last call in self.last."""

    def __init__(self, desc):
        self.d = desc

    def _in(self, a, off):
        t = torch.empty(a.size + off + 64, device="cuda")
        t[off:off + a.size] = torch.from_numpy(np.ascontiguousarray(a, np.float32).reshape(-1)).cuda()
        return t, t[off:].data_ptr()

    def _ws(self, op):
        need = self.d.workspace_bytes(op)
        ws = torch.full((need,), 0xFF, dtype=torch.uint8, device="cuda") if need else None
        return ws, need

    def call(self, op, a, b, w, bias=None, init=None, off=0, shape=None):
        """op on (a, b): forward (x, -), backward_data (dy, -), backward_filter (x, dy) with filter w; init: dw0"""
        L = capi.lib()
        ws, need = self._ws(op)
        A, pa = self._in(a, off)
        W, pw = self._in(w, 0)
        keep = [A, W]                   # the device inputs live until the output is read back
        out = Guarded(int(np.prod(shape)), off, init)
        st = capi._stream()
        if op == capi.OP_FORWARD:
            Bt, pb = self._in(bias, 0) if bias is not None else (None, 0)
            keep.append(Bt)
            rc = L.b2c_conv_forward(self.d._h, vp(pa), vp(pw), vp(pb), out.ptr(), vp(dptr(ws)), C.c_size_t(need), st)
            self.last = dict(x=pa, w=pw, y=out.ptr().value, ws=dptr(ws))
        elif op == capi.OP_BACKWARD_DATA:
            rc = L.b2c_conv_backward_data(self.d._h, vp(pa), vp(pw), out.ptr(), vp(dptr(ws)), C.c_size_t(need), st)
            self.last = dict(dy=pa, w=pw, dx=out.ptr().value, ws=dptr(ws))
        else:
            Dy, pd = self._in(b, off)
            keep.append(Dy)
            rc = L.b2c_conv_backward_filter(self.d._h, vp(pa), vp(pd), out.ptr(), vp(dptr(ws)), C.c_size_t(need), st)
            self.last = dict(x=pa, dy=pd, dw=out.ptr().value, ws=dptr(ws))
        capi.check(rc)
        return out.read().reshape(shape).copy()


def tensors(rng, po):
    x = rng.standard_normal(po.x_shape()).astype(np.float32)
    w = (rng.standard_normal(po.w_shape()) * (2.0 / po.Kd) ** 0.5).astype(np.float32)
    b = rng.standard_normal(po.O).astype(np.float32) if po.has_bias else None
    dy = rng.standard_normal(po.y_shape()).astype(np.float32)
    dw0 = rng.standard_normal(po.w_shape()).astype(np.float32)
    return x, w, b, dy, dw0


def ints(rng, shape, lim=4):
    return rng.integers(-lim, lim + 1, shape).astype(np.float32)


# ---- float64 yardsticks and the bounds of tests/test_conv_ffma_cpu.py -------------------------------------------------------------
def nobias(po):
    return o.ConvParams.make(po.N, po.C, po.H, po.W, po.O, (po.kh, po.kw), (po.sh, po.sw), (po.ph, po.pw), (po.dh, po.dw), po.G, False)


def f64_fwd(po, x, w, b):
    """(ref, magnitude): float64 forward of the oracle, the bias added in float64"""
    q = nobias(po)
    ref = o.conv_forward(q, x, w, acc64=True).astype(np.float64)
    mag = o.conv_forward(q, np.abs(x), np.abs(w), acc64=True).astype(np.float64) * SLACK
    if b is not None:
        ref += b[None, :, None, None]
        mag += np.abs(b)[None, :, None, None]
    return ref, mag


def f64_dx(po, w, dy):
    q = nobias(po)
    z = np.zeros(po.x_shape(), np.float32)
    ref = o.conv_backward(q, z, w, dy, acc64=True)[2].astype(np.float64)
    mag = o.conv_backward(q, z, np.abs(w), np.abs(dy), acc64=True)[2].astype(np.float64) * SLACK
    return ref, mag


def f64_dw(po, x, dy, dw0):
    q = nobias(po)
    z = np.zeros(po.w_shape(), np.float32)
    ref = o.conv_backward(q, x, z, dy, dw=dw0, want_dx=False, acc64=True)[0].astype(np.float64)
    mag = o.conv_backward(q, np.abs(x), z, np.abs(dy), dw=np.abs(dw0), want_dx=False, acc64=True)[0].astype(np.float64) * SLACK
    return ref, mag


def ffma_bound(po, op):
    """the factor on the magnitude: the kernel's depth plus the float64 leg's own rounding (test_conv_ffma_cpu.py)"""
    taps = po.kh * po.kw
    if op == "fwd":
        return gamma(po.Kd + 1) + U
    if op == "dgrad":
        return gamma(taps * (po.O // po.G)) + gamma(taps + 1)
    return gamma(-(-po.N * po.Ho * po.Wo // 256) + 14) + gamma(po.N)


WORST = {}


def note_worst(route, got, ref, bnd):
    r = float(np.max(np.abs(got - ref) / np.maximum(bnd, 1e-300)))
    e = rel_err(got, ref)
    w = WORST.setdefault(route, [0.0, 0.0])
    w[0], w[1] = max(w[0], e), max(w[1], r)
    print(f"[conv-ffma] route {route}: blob err {e:.3g} (worst so far {w[0]:.3g}), err / bound {r:.3g} (worst {w[1]:.3g})")


# ================================================================================================================================
# FFMA kernels
# ================================================================================================================================
S = capi.ALGO_SIMT
# (id, shape (a function of the SM count), algo, the ops checked: each must plan "simt")
FFMA_CASES = [
    # natural fallbacks: the strided Inception-v2 layers (bottoms of 28x28 and 14x14, batch reduced) ...
    ("inception_3c_3x3_dgrad", lambda S_: conv(2, 128, 28, 28, 160, 3, s=2, p=1, bias=False), None, ("dgrad",)),
    ("inception_3c_5x5b_dgrad", lambda S_: conv(2, 64, 28, 28, 96, 5, s=2, p=2, bias=False), None, ("dgrad",)),
    ("inception_4e_3x3_dgrad", lambda S_: conv(2, 128, 14, 14, 192, 3, s=2, p=1, bias=False), None, ("dgrad",)),
    ("inception_4e_5x5b_dgrad", lambda S_: conv(2, 192, 14, 14, 256, 5, s=2, p=2, bias=False), None, ("dgrad",)),
    # ... the gather-table cliffs (K / 4 > 1152 chunks in KMODE 1, K > 1152 in KMODE 0, Og past the dgrad table) ...
    ("fwd_cliff_kmode1_k4644", lambda S_: conv(1, 516, 5, 5, 32, 3, s=2, p=1), None, ("fwd",)),
    ("fwd_cliff_kmode0_k1161", lambda S_: conv(1, 129, 5, 5, 32, 3, s=2, p=1), None, ("fwd",)),
    ("dgrad_cliff_og516", lambda S_: conv(1, 8, 4, 4, 1032, 3, p=1, G=2, bias=False), None, ("dgrad",)),
    # ... the 7x7/s2 stem and a 3x3/s2 layer with odd W
    ("stem_7x7_s2_dgrad", lambda S_: conv(1, 3, 224, 224, 64, 7, s=2, p=3, bias=False), None, ("dgrad",)),
    ("dgrad_3x3_s2_odd_w", lambda S_: conv(2, 36, 13, 13, 64, 3, s=2, p=1), None, ("dgrad",)),
    # ALGO_SIMT: every op
    ("simt_group2", lambda S_: conv(2, 8, 9, 9, 6, 3, p=1, G=2), S, ("fwd", "dgrad", "wgrad")),
    ("simt_group3_cg3", lambda S_: conv(2, 9, 9, 9, 12, 3, p=1, G=3), S, ("fwd", "dgrad", "wgrad")),
    ("simt_dilation2", lambda S_: conv(2, 6, 12, 12, 8, 3, p=2, d=2), S, ("fwd", "dgrad", "wgrad")),
    ("simt_pad_ge_k", lambda S_: conv(2, 3, 5, 5, 4, 3, p=3), S, ("fwd", "dgrad", "wgrad")),
    ("simt_1x7", lambda S_: conv(2, 5, 9, 17, 6, (1, 7), p=(0, 3)), S, ("fwd", "dgrad", "wgrad")),
    ("simt_7x1", lambda S_: conv(2, 5, 17, 9, 6, (7, 1), p=(3, 0)), S, ("fwd", "dgrad", "wgrad")),
    ("simt_stride_2x3", lambda S_: conv(2, 4, 13, 17, 6, 3, s=(2, 3), p=1), S, ("fwd", "dgrad", "wgrad")),
    ("simt_1x1_s2", lambda S_: conv(2, 16, 9, 9, 8, 1, s=2, bias=False), S, ("fwd", "dgrad", "wgrad")),
    ("simt_1x1_maps_k1", lambda S_: conv(3, 8, 1, 1, 10, 1), S, ("fwd", "dgrad", "wgrad")),
    ("simt_1x1_maps_k3_p1", lambda S_: conv(3, 8, 1, 1, 10, 3, p=1), S, ("fwd", "dgrad", "wgrad")),
    # N * O * Ho * Wo and N * C * H * W above sm_count * 16 * 256: the grid strides
    ("simt_grid_strides", lambda S_: conv(-(-S_ * 16 * 256 // (40 * 64 * 64)) + 1, 40, 64, 64, 40, 3, p=1), S,
     ("fwd", "dgrad", "wgrad")),
    # weight gradient: Q = N * Ho * Wo < 32, not a multiple of 256, 2 / 3 / 4 multiples of 256; Cg > 1 with G > 1 above
    ("wgrad_q4", lambda S_: conv(1, 4, 4, 4, 3, 3), S, ("wgrad",)),
    ("wgrad_q338", lambda S_: conv(2, 4, 13, 13, 5, 3, p=1), S, ("wgrad",)),
    ("wgrad_q512", lambda S_: conv(2, 4, 16, 16, 5, 3, p=1), S, ("wgrad",)),
    ("wgrad_q768", lambda S_: conv(3, 4, 16, 16, 5, 3, p=1), S, ("wgrad",)),
    ("wgrad_q1024_g2", lambda S_: conv(4, 6, 16, 16, 4, 3, p=1, G=2), S, ("wgrad",)),
]
FFMA_IDS = [c[0] for c in FFMA_CASES]


def route_of(desc, op):
    return desc.wgrad_plan()["route"] if op == "wgrad" else desc.conv_plan(OPS[op])["route"]


@pytest.mark.parametrize("cid,shape,algo,ops", FFMA_CASES, ids=FFMA_IDS)
def test_ffma_kernels_bit_exact(rng, sms, cid, shape, algo, ops):
    c = shape(sms)
    po, pc = params(o, c), params(capi, c)
    d = m.ConvDesc(pc, algo=algo)
    for op in ops:
        assert route_of(d, op) == "simt", f"{op}: the planner no longer sends this case to the FFMA kernel ({route_of(d, op)})"
        assert d.algo_used(OPS[op]) == capi.ALGO_SIMT
    if cid == "simt_grid_strides":
        assert min(po.N * po.O * po.Ho * po.Wo, po.N * po.C * po.H * po.W) > sms * 16 * 256
    x, w, b, dy, dw0 = tensors(rng, po)
    run = Caller(d)
    for op in ops:
        if op == "fwd":
            want = o.conv_fwd_ffma(po, x, w, b)
            go = lambda off: run.call(capi.OP_FORWARD, x, None, w, b, off=off, shape=po.y_shape())
            ref, mag = f64_fwd(po, x, w, b)
        elif op == "dgrad":
            want = o.conv_dgrad_ffma(po, w, dy)
            go = lambda off: run.call(capi.OP_BACKWARD_DATA, dy, None, w, off=off, shape=po.x_shape())
            ref, mag = f64_dx(po, w, dy)
        else:
            want = o.conv_wgrad_ffma(po, x, dy, dw0)
            go = lambda off: run.call(capi.OP_BACKWARD_FILTER, x, dy, w, init=dw0, off=off, shape=po.w_shape())
            ref, mag = f64_dw(po, x, dy, dw0)
        got = go(0)
        assert_bits(got, want, f"{op} against its restatement")
        assert_bits(go(0), got, f"{op}, second call")
        assert_bits(go(1), got, f"{op}, operands 4 bytes off alignment")
        bnd = ffma_bound(po, op) * mag
        bad = np.argwhere(np.abs(got - ref) > bnd)
        assert bad.size == 0, f"{op}: {len(bad)} elements outside the float64 bound, first at {tuple(bad[0])}"
        note_worst("simt " + op, got, ref, bnd)


# ================================================================================================================================
# CAFFE engine
# ================================================================================================================================
# (id, shape, the route of the per-image weight-gradient GEMMs); N >= 3 so the col buffer is reused
CAFFE_CASES = [
    ("caffe_3x3_p1_8x8", conv(3, 8, 8, 8, 12, 3, p=1), "tc"),                 # P = 64
    ("caffe_3x3_p1_7x7", conv(3, 8, 7, 7, 12, 3, p=1), "ffma"),               # P = 49
    ("caffe_strided_13x13", conv(3, 6, 13, 13, 10, 3, s=2, p=1), "ffma"),     # 7x7 out
    ("caffe_dilated_13x13", conv(3, 5, 13, 13, 7, 3, p=2, d=2), "ffma"),      # P = 169
    ("caffe_group2_og70", conv(3, 8, 13, 13, 140, 3, p=1, G=2), "ffma"),
    ("caffe_group2_og70_8x8", conv(3, 8, 8, 8, 140, 3, p=1, G=2), "tc"),
    ("caffe_1x1_7x7", conv(3, 16, 7, 7, 24, 1), "ffma"),                      # workspace 0: a null pointer
    ("caffe_1x1_8x8", conv(3, 16, 8, 8, 24, 1, bias=False), "tc"),
]
CAFFE_IDS = [c[0] for c in CAFFE_CASES]


def is_1x1(po):
    return po.kh == po.kw == 1 and po.sh == po.sw == 1 and po.ph == po.pw == 0


def im2col_of(po, img):
    return o.im2col(img, (po.kh, po.kw), (po.sh, po.sw), (po.ph, po.pw), (po.dh, po.dw)).reshape(po.Kd * po.G, -1)


def caffe_gemm_plans(po, last, op):
    """the sgemm_plan of every GEMM the CAFFE engine issues for `op`, at the pointers of the call"""
    P, Og, Kd, F = po.Ho * po.Wo, po.O // po.G, po.Kd, 4
    bdim, tdim = po.C * po.H * po.W, po.O * P
    plans = []
    for n in range(po.N):
        for g in range(po.G):
            if op == "fwd":
                B = (last["x"] + F * n * bdim if is_1x1(po) else last["ws"]) + F * g * Kd * P
                plans.append(capi.sgemm_plan(0, 0, Og, P, Kd, 1.0, 0.0, last["w"] + F * g * Og * Kd, B))
            elif op == "dgrad":
                plans.append(capi.sgemm_plan(1, 0, Kd, P, Og, 1.0, 0.0, last["w"] + F * g * Og * Kd, last["dy"] + F * (n * tdim + g * Og * P)))
            else:
                B = (last["x"] + F * n * bdim if is_1x1(po) else last["ws"]) + F * g * Kd * P
                plans.append(capi.sgemm_plan(0, 1, Og, Kd, P, 1.0, 1.0, last["dy"] + F * (n * tdim + g * Og * P), B))
    return plans


def caffe_fwd(po, x, w, b):
    P, Og, Kd = po.Ho * po.Wo, po.O // po.G, po.Kd
    y = np.empty((po.N, po.O, P), np.float32)
    for n in range(po.N):
        col = x[n].reshape(po.C, P) if is_1x1(po) else im2col_of(po, x[n])
        for g in range(po.G):
            y[n, g * Og:(g + 1) * Og] = o.gemm_ffma(0, 0, Og, P, Kd, 1.0, w[g * Og:(g + 1) * Og].reshape(Og, Kd),
                                                    col[g * Kd:(g + 1) * Kd], 0.0, np.zeros((Og, P), np.float32))[0]
    if b is not None:
        y = y + b[None, :, None]                                  # bias_add_kernel: one fp32 add per element
    return y.reshape(po.y_shape())


def caffe_dx(po, w, dy):
    P, Og, Kd = po.Ho * po.Wo, po.O // po.G, po.Kd
    dx = np.empty(po.x_shape(), np.float32)
    for n in range(po.N):
        col = np.concatenate([o.gemm_ffma(1, 0, Kd, P, Og, 1.0, w[g * Og:(g + 1) * Og].reshape(Og, Kd),
                                          dy[n, g * Og:(g + 1) * Og].reshape(Og, P), 0.0, np.zeros((Kd, P), np.float32))[0]
                              for g in range(po.G)])
        # the 1x1 shortcut writes the GEMM straight into dx (col2im would turn a -0 into +0)
        dx[n] = col.reshape(po.C, po.H, po.W) if is_1x1(po) else o.col2im(col, (po.C, po.H, po.W), (po.kh, po.kw), (po.sh, po.sw),
                                                                         (po.ph, po.pw), (po.dh, po.dw))
    return dx


def caffe_dw_forms(po, x, dy, dw0):
    """N = 1: the three admissible results of the one NT GEMM per group with beta = 1"""
    assert po.N == 1
    P, Og, Kd = po.Ho * po.Wo, po.O // po.G, po.Kd
    col = x[0].reshape(po.C, P) if is_1x1(po) else im2col_of(po, x[0])
    out = np.empty((3, po.O, Kd), np.float32)
    for g in range(po.G):
        out[:, g * Og:(g + 1) * Og] = o.gemm_ffma(0, 1, Og, Kd, P, 1.0, dy[0, g * Og:(g + 1) * Og].reshape(Og, P),
                                                  col[g * Kd:(g + 1) * Kd], 1.0, dw0[g * Og:(g + 1) * Og].reshape(Og, Kd))
    return out.reshape((3,) + po.w_shape())


def per_image_dw(po, x, dy):
    """float64 [N, O, Kd] per-image products and their magnitudes"""
    P, Og, Kd = po.Ho * po.Wo, po.O // po.G, po.Kd
    prods, mags = np.zeros((po.N, po.O, Kd)), np.zeros((po.N, po.O, Kd))
    for n in range(po.N):
        col = (x[n].reshape(po.C, P) if is_1x1(po) else im2col_of(po, x[n])).astype(np.float64)
        for g in range(po.G):
            a = dy[n, g * Og:(g + 1) * Og].reshape(Og, P).astype(np.float64)
            bcol = col[g * Kd:(g + 1) * Kd]
            prods[n, g * Og:(g + 1) * Og] = a @ bcol.T
            mags[n, g * Og:(g + 1) * Og] = np.abs(a) @ np.abs(bcol).T
    return prods, mags


def chained_dw_bound(po, plans, prods, mags, dw0, calls=1):
    """(ref, bound) of dW after `calls` weight-gradient calls of N per-image beta = 1 GEMMs from dw0.  An FFMA GEMM is a chain of
    16 ceil(P / 16) fmaf steps plus the two roundings of the store; a tensor-core one is bounded per element as in
    tests/test_gemm_schedule_gpu.py (tc_bound); per-call errors add."""
    ref = dw0.reshape(po.O, -1).astype(np.float64).copy()
    bnd = np.zeros_like(ref)
    q = plans[0]
    for _ in range(calls):
        for n in range(po.N):
            prev = np.abs(ref)
            ref += prods[n]
            if q["route"] == "ffma":
                kp = 16 * -(-(po.Ho * po.Wo) // 16)
                bnd += gamma(kp + 2) * (mags[n] + prev + np.abs(ref))
            else:
                k = 12 * q["kb_per_split"] + q["splits"] + 1
                bnd += (2.0 ** -16 + k * 2.0 ** -23) * mags[n] + 2.0 ** -24 * np.abs(ref) + 2.0 ** -23 * np.abs(ref)
    return ref, bnd * SLACK


@pytest.mark.parametrize("cid,c,wroute", CAFFE_CASES, ids=CAFFE_IDS)
def test_caffe_engine(rng, cid, c, wroute):
    po, pc = params(o, c), params(capi, c)
    d = m.ConvDesc(pc, capi.ENGINE_CAFFE)
    assert d.conv_plan(capi.OP_FORWARD)["route"] == d.conv_plan(capi.OP_BACKWARD_DATA)["route"] == "caffe"
    assert d.wgrad_plan()["route"] == "caffe"
    for op in OPS.values():
        assert d.workspace_bytes(op) == (0 if is_1x1(po) else 4 * po.Kd * po.G * po.Ho * po.Wo)
    x, w, b, dy, dw0 = tensors(rng, po)
    run = Caller(d)
    # forward
    y = run.call(capi.OP_FORWARD, x, None, w, b, shape=po.y_shape())
    assert all(q["route"] == "ffma" for q in caffe_gemm_plans(po, run.last, "fwd"))
    assert_bits(y, caffe_fwd(po, x, w, b), "forward against im2col + FFMA GEMM + bias")
    assert_bits(run.call(capi.OP_FORWARD, x, None, w, b, shape=po.y_shape()), y, "forward, second call")
    ref, mag = f64_fwd(po, x, w, b)
    note_worst("caffe fwd", y, ref, gamma(16 * -(-po.Kd // 16) + 2) * mag)
    # data gradient
    dx = run.call(capi.OP_BACKWARD_DATA, dy, None, w, shape=po.x_shape())
    assert all(q["route"] == "ffma" for q in caffe_gemm_plans(po, run.last, "dgrad"))
    assert_bits(dx, caffe_dx(po, w, dy), "data gradient against FFMA GEMM + col2im")
    assert_bits(run.call(capi.OP_BACKWARD_DATA, dy, None, w, shape=po.x_shape()), dx, "data gradient, second call")
    ref, mag = f64_dx(po, w, dy)
    taps = po.kh * po.kw
    note_worst("caffe dgrad", dx, ref, (gamma(16 * -(-(po.O // po.G) // 16) + 2 + taps) + gamma(taps + 1)) * mag)
    # weight gradient, float data
    dw = run.call(capi.OP_BACKWARD_FILTER, x, dy, w, init=dw0, shape=po.w_shape())
    plans = caffe_gemm_plans(po, run.last, "wgrad")
    assert all(q["route"] == wroute for q in plans), (wroute, plans)
    assert_bits(run.call(capi.OP_BACKWARD_FILTER, x, dy, w, init=dw0, shape=po.w_shape()), dw, "weight gradient, second call")
    prods, mags = per_image_dw(po, x, dy)
    ref, bnd = chained_dw_bound(po, plans, prods, mags, dw0)
    got = dw.reshape(po.O, -1)
    bad = np.argwhere(np.abs(got - ref) > bnd)
    assert bad.size == 0, f"weight gradient ({wroute}): {len(bad)} elements outside the bound, first at {tuple(bad[0])}"
    note_worst(f"caffe wgrad ({wroute})", got, ref, bnd)
    # weight gradient, integer data: exact whatever the contraction or the order
    xi, dyi, dwi = ints(rng, po.x_shape()), ints(rng, po.y_shape()), ints(rng, po.w_shape())
    got = run.call(capi.OP_BACKWARD_FILTER, xi, dyi, w, init=dwi, shape=po.w_shape())
    want = dwi.reshape(po.O, -1).astype(np.float64) + per_image_dw(po, xi, dyi)[0].sum(0)
    assert np.abs(want).max() < 2 ** 24
    assert_bits(got.reshape(po.O, -1), want.astype(np.float32), "weight gradient on integer data")
    # one image: one NT GEMM per group, bit for bit when it runs on the FFMA kernel
    if wroute == "ffma":
        p1, c1 = params(o, c, N=1), params(capi, c, N=1)
        run1 = Caller(m.ConvDesc(c1, capi.ENGINE_CAFFE))
        got = run1.call(capi.OP_BACKWARD_FILTER, x[:1], dy[:1], w, init=dw0, shape=p1.w_shape())
        assert all(q["route"] == "ffma" for q in caffe_gemm_plans(p1, run1.last, "wgrad"))
        ok = o.ffma_match(got, caffe_dw_forms(p1, x[:1], dy[:1], dw0))
        assert ok.all(), f"weight gradient, N = 1: {int((~ok).sum())} elements match no admissible FFMA result"


@pytest.mark.parametrize("math,algo", [(capi.MATH_FP32, capi.ALGO_AUTO), (capi.MATH_TF32, capi.ALGO_TCGEN05),
                                       (capi.MATH_FP32_3XTF32, capi.ALGO_SIMT)], ids=["fp32_auto", "tf32_tc", "3xtf32_simt"])
def test_caffe_engine_reports_simt_whatever_the_descriptor_asks(math, algo):
    c = CAFFE_CASES[0][1]
    d = m.ConvDesc(params(capi, c), capi.ENGINE_CAFFE, math=math, algo=algo)
    for op in OPS.values():
        assert d.algo_used(op) == capi.ALGO_SIMT
    assert d.conv_plan(capi.OP_FORWARD)["route"] == "caffe" and d.wgrad_plan()["route"] == "caffe"


# ================================================================================================================================
# N-D path of the host layer
# ================================================================================================================================
# (id, bottom shape, num_output, kernel, stride, pad, dilation, group, force_nd)
ND_CASES = [
    ("simple_3d", (2, 3, 5, 6, 4), 4, (3, 3, 3), (2, 2, 2), (0, 0, 0), (1, 1, 1), 1, False),      # TestSimple3DConvolution
    ("grouped_3d", (3, 4, 4, 5, 6), 6, (2, 3, 3), (1, 1, 1), (1, 1, 1), (1, 1, 1), 2, False),
    ("per_axis_3d", (2, 3, 6, 7, 5), 5, (3, 2, 3), (2, 1, 1), (1, 0, 1), (1, 2, 1), 1, False),
    ("force_nd_2d_s2", (3, 4, 9, 7), 5, (3, 3), (2, 2), (1, 1), (1, 1), 1, True),
    ("force_nd_2d_g2_8x8", (3, 6, 8, 8), 4, (3, 3), (1, 1), (1, 1), (1, 1), 2, True),                # P = 64: dW on the tensor cores
]
ND_IDS = [c[0] for c in ND_CASES]
ALIGNED_BASE = 1 << 20


def nd_geometry(shape, O, k, s, p, d, G):
    out = tuple((shape[2 + a] + 2 * p[a] - (d[a] * (k[a] - 1) + 1)) // s[a] + 1 for a in range(len(k)))
    Kd = shape[1] // G * int(np.prod(k))
    return out, int(np.prod(out)), Kd


def nd_plans(shape, O, k, s, p, d, G):
    """the GEMM plans of the layer's calls, at a 256-byte aligned base plus each call's offsets"""
    out, P, Kd = nd_geometry(shape, O, k, s, p, d, G)
    N, Og, F, B = shape[0], O // G, 4, ALIGNED_BASE
    tdim = O * P
    plans = {"fwd": [], "bias": [], "dgrad": [], "wgrad": []}
    for n in range(N):
        for g in range(G):
            plans["fwd"].append(capi.sgemm_plan(0, 0, Og, P, Kd, 1.0, 0.0, B + F * g * Og * Kd, B + F * g * Kd * P))
            plans["dgrad"].append(capi.sgemm_plan(1, 0, Kd, P, Og, 1.0, 0.0, B + F * g * Og * Kd, B + F * (n * tdim + g * Og * P)))
            plans["wgrad"].append(capi.sgemm_plan(0, 1, Og, Kd, P, 1.0, 1.0, B + F * (n * tdim + g * Og * P), B + F * g * Kd * P))
        plans["bias"].append(capi.sgemm_plan(0, 0, O, P, 1, 1.0, 1.0, B, B))
    return plans


def nd_y(x, w, b, O, k, s, p, d, G):
    N = x.shape[0]
    out, P, Kd = nd_geometry(x.shape, O, k, s, p, d, G)
    Og = O // G
    y = np.empty((N, O, P), np.float32)
    for n in range(N):
        col = o.im2col_nd(x[n], k, s, p, d).reshape(Kd * G, P)
        for g in range(G):
            y[n, g * Og:(g + 1) * Og] = o.gemm_ffma(0, 0, Og, P, Kd, 1.0, w[g * Og:(g + 1) * Og].reshape(Og, Kd),
                                                    col[g * Kd:(g + 1) * Kd], 0.0, np.zeros((Og, P), np.float32))[0]
    forms = np.stack([o.gemm_ffma(0, 0, O, P, 1, 1.0, b.reshape(O, 1), np.ones((1, P), np.float32), 1.0, y[n]) for n in range(N)], 1)
    return forms.reshape((3, N, O) + out)


def nd_dx(x_shape, w, dy, O, k, s, p, d, G):
    N = x_shape[0]
    out, P, Kd = nd_geometry(x_shape, O, k, s, p, d, G)
    Og = O // G
    dx = np.empty(x_shape, np.float32)
    for n in range(N):
        col = np.concatenate([o.gemm_ffma(1, 0, Kd, P, Og, 1.0, w[g * Og:(g + 1) * Og].reshape(Og, Kd),
                                          dy[n, g * Og:(g + 1) * Og].reshape(Og, P), 0.0, np.zeros((Kd, P), np.float32))[0]
                              for g in range(G)])
        dx[n] = o.col2im_nd(col.reshape((Kd * G,) + out), x_shape[1:], k, s, p, d)
    return dx


def nd_layer(shape, O, k, s, p, d, G, force, w, b):
    L = h.ConvolutionLayer(O, k, s, p, d, G, True, capi.ENGINE_CAFFE, force_nd=force)
    L.setup(shape)
    L.set_blob(0, w)
    L.set_blob(1, b)
    return L


def nd_dw_db_f64(x, dy, dw0, db0, O, k, s, p, d, G, calls):
    """float64 (dW, its bound magnitude per image, db) pieces for chained_dw_bound-like checks"""
    N = x.shape[0]
    out, P, Kd = nd_geometry(x.shape, O, k, s, p, d, G)
    Og = O // G
    prods, mags = np.zeros((N, O, Kd)), np.zeros((N, O, Kd))
    for n in range(N):
        col = o.im2col_nd(x[n], k, s, p, d).reshape(Kd * G, P).astype(np.float64)
        for g in range(G):
            a = dy[n, g * Og:(g + 1) * Og].reshape(Og, P).astype(np.float64)
            prods[n, g * Og:(g + 1) * Og] = a @ col[g * Kd:(g + 1) * Kd].T
            mags[n, g * Og:(g + 1) * Og] = np.abs(a) @ np.abs(col[g * Kd:(g + 1) * Kd]).T
    dyf = dy.reshape(N, O, P).astype(np.float64)
    db_ref = db0.astype(np.float64) + calls * dyf.sum((0, 2))
    # sgemv NoTrans per image: 32 lane chains of ceil(P / 32), 5 butterfly adds, the store's two roundings
    db_bnd = gamma(calls * N * (-(-P // 32) + 7)) * (np.abs(db0) + calls * np.abs(dyf).sum((0, 2))) * SLACK
    return prods, mags, db_ref, db_bnd, P, Kd


class _NDPrm:
    """the fields chained_dw_bound reads, for an N-D layer"""

    def __init__(self, N, O, P):
        self.N, self.O, self.G, self.Ho, self.Wo = N, O, 1, 1, P


@pytest.mark.parametrize("cid,shape,O,k,s,p,d,G,force", ND_CASES, ids=ND_IDS)
def test_nd_layer(rng, cid, shape, O, k, s, p, d, G, force):
    plans = nd_plans(shape, O, k, s, p, d, G)
    assert all(q["route"] == "ffma" for key in ("fwd", "bias", "dgrad") for q in plans[key])
    wr = {q["route"] for q in plans["wgrad"]}
    assert len(wr) == 1
    out, P, Kd = nd_geometry(shape, O, k, s, p, d, G)
    assert wr == ({"tc"} if P >= 64 and P % 4 == 0 else {"ffma"}), (wr, P)
    wshape = (O, shape[1] // G) + tuple(k)
    yshape = (shape[0], O) + out
    for data in ("float", "int"):
        if data == "float":
            x, dy = rng.standard_normal(shape).astype(np.float32), rng.standard_normal(yshape).astype(np.float32)
            w = (rng.standard_normal(wshape) * 0.3).astype(np.float32)
            b, db0 = rng.standard_normal(O).astype(np.float32), rng.standard_normal(O).astype(np.float32)
            dw0 = rng.standard_normal(wshape).astype(np.float32)
        else:
            x, dy, w, b, db0, dw0 = (ints(rng, s_) for s_ in (shape, yshape, wshape, (O,), (O,), wshape))
        L = nd_layer(shape, O, k, s, p, d, G, force, w, b)
        L.set_blob(0, dw0, diff=True)
        L.set_blob(1, db0, diff=True)
        y = L.forward(x)
        ok = o.ffma_match(y, nd_y(x, w, b, O, k, s, p, d, G))
        assert ok.all(), f"{data}: y: {int((~ok).sum())} elements match no admissible im2col_nd + GEMM + bias GEMM result"
        want_dx = nd_dx(shape, w, dy, O, k, s, p, d, G)
        dx = L.backward(dy)
        assert_bits(dx, want_dx, f"{data}: dx against FFMA GEMM TN + col2im_nd")
        assert_bits(L.backward(dy), want_dx, f"{data}: dx of the second Backward (overwritten, not accumulated)")
        dw, db = L.get_blob(0, True).reshape(O, -1), L.get_blob(1, True)
        prods, mags, db_ref, db_bnd, _, _ = nd_dw_db_f64(x, dy, dw0, db0, O, k, s, p, d, G, 2)
        if data == "int":
            want = dw0.reshape(O, -1).astype(np.float64) + 2 * prods.sum(0)
            assert np.abs(want).max() < 2 ** 24
            assert_bits(dw, want.astype(np.float32), "int: dW after two Backward calls")
            assert_bits(db, db_ref.astype(np.float32), "int: db after two Backward calls")
            continue
        ref, bnd = chained_dw_bound(_NDPrm(shape[0], O, P), plans["wgrad"], prods, mags, dw0, calls=2)
        bad = np.argwhere(np.abs(dw - ref) > bnd)
        assert bad.size == 0, f"dW after two Backward calls: {len(bad)} elements outside the bound, first at {tuple(bad[0])}"
        assert (np.abs(db - db_ref) <= db_bnd).all(), "db after two Backward calls outside the bound"
        note_worst("nd wgrad (" + next(iter(wr)) + ")", dw, ref, bnd)
    # one image, one Backward: the dW GEMM per group and the db GEMV bit for bit against their admissible results
    shape1 = (1,) + tuple(shape[1:])
    x1 = rng.standard_normal(shape1).astype(np.float32)
    dy1 = rng.standard_normal((1, O) + out).astype(np.float32)
    L = nd_layer(shape1, O, k, s, p, d, G, force, w, b)
    L.set_blob(0, dw0, diff=True)
    L.set_blob(1, db0, diff=True)
    L.forward(x1)
    L.backward(dy1)
    db_forms = o.gemv_ffma(0, O, P, 1.0, dy1.reshape(O, P), np.ones(P, np.float32), 1.0, db0)
    ok = o.ffma_match(L.get_blob(1, True), db_forms)
    assert ok.all(), f"db, one image: {int((~ok).sum())} elements match no admissible GEMV result"
    if wr == {"ffma"}:
        col = o.im2col_nd(x1[0], k, s, p, d).reshape(Kd * G, P)
        Og = O // G
        forms = np.concatenate([o.gemm_ffma(0, 1, Og, Kd, P, 1.0, dy1[0, g * Og:(g + 1) * Og].reshape(Og, P), col[g * Kd:(g + 1) * Kd],
                                            1.0, dw0[g * Og:(g + 1) * Og].reshape(Og, Kd)) for g in range(G)], 1)
        ok = o.ffma_match(L.get_blob(0, True).reshape(O, Kd), forms)
        assert ok.all(), f"dW, one image: {int((~ok).sum())} elements match no admissible FFMA GEMM result"


def test_worst_errors_reported():
    """prints the worst blob error and err / bound per route over the cases that ran before it"""
    for route, (e, r) in sorted(WORST.items()):
        print(f"[conv-ffma] worst over the suite, {route}: blob err {e:.3g}, err / bound {r:.3g}")
        assert r <= 1.0

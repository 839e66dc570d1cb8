"""The GEMM family behind b2c_sgemm / b2c_sgemm_ex / b2c_sgemv, element by element, on every launch regime.

b2c_sgemm_ex runs one of two kernels (include/b2c.h, b2c_sgemm_route): the staged bf16x3 tensor-core kernel for NoTrans x Trans
products with alpha = 1, beta in {0, 1}, K >= 64, K % 4 == 0, 16-byte aligned operands and the default fp32 math, split over one
wave of CTAs when the caller brings a workspace (without one, a product the planner would split runs unsplit, and on the FFMA
kernel past 256 K blocks of 64); and the FFMA kernel for everything else.  Every case asserts its regime on
capi.sgemm_plan() (b2c_debug_sgemm_plan, the planner the launch runs), so a planner change that moves a case off its path fails
here, naming the regime.  Shapes that depend on the split plan are scaled by the device's SM count.

What each route is held to:
  * FFMA GEMM and both GEMV kernels: bit for bit against oracle.gemm_ffma / gemv_ffma, which restate their fmaf chains (the GEMV's
    lane-strided chains and xor butterfly included); an element may equal any of the three contractions of alpha * acc + beta * c.
    A wrong leading dimension, transpose loader or tile-edge / K-tail index moves bits, however small the element.
  * tensor cores, integer data (|a|, |b| <= 8: exact in bf16, so every lo part is 0 and every partial sum an integer below 2^24):
    equal to the float64 product, bit for bit.  A term dropped or counted twice at a K tail, a tile edge or a split boundary shows.
  * tensor cores, float data: per element  |got - ref| <= (2^-16 + n * 2^-23) * sum_k |a_k b_k| + 2^-24 |ref|.
    split_pack_bf16 keeps a = hi + lo + r with |a - hi| <= 2^-9 |a| and |r| <= 2^-9 |a - hi| <= 2^-18 |a|; the three MMAs
    hi*hi + hi*lo + lo*hi miss lo*lo and the r terms, at most 3 * 2^-18 |ab| (+ O(2^-27)) < 2^-16 |ab| per product.  Each
    product of a bf16 pair is exact in fp32.  The fp32 accumulator takes n additions -- 3 MMAs per 16-wide K step over the
    CTA's kb_per_split blocks of 64 (12 per block), then one per split in the fixed-order reduction and one for beta * C -- each
    off by at most one unit in the last place (2^-23 relative, whatever the adder's rounding) of a partial sum bounded by
    sum |ab|.  The last term is the final rounding.  Rows of A and B are scaled by different powers of two so that sum |ab|
    spans decades across the output: the bound is tight where the values are small.  The suites' 1e-4 blob bar applies too.

Harness (as test_wgrad_schedule_gpu.py): C is a view between sentinel guard bands; the workspace is NaN; with beta = 0, C starts
as NaN and none may leak; a second call (workspace refilled with other bytes) gives the same bits; beta = 1 with A = 0 leaves C
bit-identical to C0.  InnerProduct is also run whole through TrainNet at batches that reach its tensor-core backward."""
import ctypes as C
import os

import numpy as np
import pytest

import oracle as o
from cases import rel_err

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from caffe_mpi_b200 import capi, host_api, models  # noqa: E402

TOL = 1e-4
GUARD = 64                                   # sentinel floats before and after C (256 bytes: C stays 16-byte aligned)
SENTINEL = np.float32(-7.25e19)


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def host(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.int32)


def operand(a, off):
    """a on the device at element offset `off` inside its buffer (off = 1: 4-byte aligned only)"""
    buf = torch.empty(max(a.size, 1) + off, device="cuda")       # K = 0 still passes a non-null pointer
    buf[off:off + a.size] = dev(a.reshape(-1))
    return buf[off:]


class Gemm:
    """One b2c_sgemm_ex call through the C ABI.  ws: "planned" (b2c_sgemm_workspace_bytes, NaN-filled), None, "short" (4 bytes
    less) or "misaligned" (the planned size at a 4-byte offset).  a_off / b_off / c_off: element offsets of A, B and C."""

    def __init__(self, tA, tB, M, N, K, alpha, beta, a, b, ws="planned", a_off=0, b_off=0, c_off=0):
        self.tA, self.tB, self.M, self.N, self.K, self.alpha, self.beta = tA, tB, M, N, K, alpha, beta
        self.A, self.B = operand(a, a_off), operand(b, b_off)
        self.c_off = c_off
        need = capi.lib().b2c_sgemm_workspace_bytes(tA, tB, M, N, K)
        self.ws_mode = ws
        if ws is None:
            self.ws_buf, self.ws_ptr, self.ws_bytes = None, 0, 0
        else:
            self.ws_buf = torch.empty(max(need, 16) + 16, dtype=torch.uint8, device="cuda")
            self.ws_ptr = self.ws_buf.data_ptr() + (4 if ws == "misaligned" else 0)
            self.ws_bytes = max(need - 4, 0) if ws == "short" else need

    def plan(self):
        return capi.sgemm_plan(self.tA, self.tB, self.M, self.N, self.K, self.alpha, self.beta, self.A.data_ptr(), self.B.data_ptr(),
                               self.ws_ptr, self.ws_bytes)

    def call(self, c0, A=None, ws_fill=0xFF):
        """C after the call (C0 = c0, or NaN when beta = 0); checks the guard bands"""
        n = self.M * self.N
        buf = torch.full((GUARD + self.c_off + n + GUARD,), float(SENTINEL), device="cuda")
        body = buf[GUARD + self.c_off:GUARD + self.c_off + n]
        if self.beta == 0.0:
            body.fill_(float("nan"))
        else:
            body.copy_(dev(c0.reshape(-1)))
        if self.ws_buf is not None:
            self.ws_buf.fill_(ws_fill)
        A = self.A if A is None else A
        L = capi.lib()
        capi.check(L.b2c_sgemm_ex(self.tA, self.tB, self.M, self.N, self.K, self.alpha, C.c_void_p(A.data_ptr()),
                                  C.c_void_p(self.B.data_ptr()), self.beta, C.c_void_p(body.data_ptr()),
                                  C.c_void_p(self.ws_ptr or None), self.ws_bytes, capi._stream()))
        out = host(buf)
        guard = np.concatenate([out[:GUARD + self.c_off], out[GUARD + self.c_off + n:]])
        assert (bits(guard) == bits(SENTINEL)).all(), "write outside C"
        return out[GUARD + self.c_off:GUARD + self.c_off + n].reshape(self.M, self.N)

    def checked(self, c0):
        """the harness: no NaN, same bits on a second call, beta = 1 with A = 0 gives C0"""
        got = self.call(c0)
        assert not np.isnan(got).any(), "NaN in C: C (beta = 0) or a workspace partial leaked"
        again = self.call(c0, ws_fill=0x5A)
        assert np.array_equal(bits(got), bits(again)), "not bit-identical run to run"
        if self.beta == 1.0:
            zero = self.call(c0, A=torch.zeros_like(self.A))
            assert np.array_equal(bits(zero), bits(c0)), "A = 0 with beta = 1 changed C"
        return got


def ffma_plan(M, N, K):
    nk = (K + 15) // 16
    return dict(route="ffma", cols=64, bpi=nk, splits=1, kb_per_split=nk, m_tiles=(M + 63) // 64, n_tiles=(N + 63) // 64)


def op_shapes(tA, tB, M, N, K):
    return ((K, M) if tA else (M, K)), ((N, K) if tB else (K, N))


def check_ffma(g, a, b, c0):
    got = g.checked(c0)
    want = o.gemm_ffma(g.tA, g.tB, g.M, g.N, g.K, g.alpha, a, b, g.beta, c0)
    ok = o.ffma_match(got, want)
    bad = np.argwhere(~ok)
    assert bad.size == 0, (f"{(~ok).sum()} of {ok.size} elements differ from the FFMA chain, first at {tuple(bad[0])}: "
                           f"got {got[tuple(bad[0])]!r}, want one of {want[:, bad[0][0], bad[0][1]]}")
    return got


# ---- FFMA route: bit-exact, every transpose pair, tile edges and K tails ----------------------------------------------------
MNS = (1, 63, 64, 65, 127, 129)
ALPHA_BETA = [(al, be) for al in (1.0, 0.5, -3.0) for be in (0.0, 1.0, -2.0)]


def goes_tc(tA, tB, K, alpha, beta):
    return (not tA) and tB and alpha == 1.0 and beta in (0.0, 1.0) and K >= 64 and K % 4 == 0


@pytest.mark.parametrize("K", [0, 1, 15, 16, 17, 100])
@pytest.mark.parametrize("tA,tB", [(0, 0), (0, 1), (1, 0), (1, 1)], ids=["NN", "NT", "TN", "TT"])
def test_ffma_bit_exact(rng, tA, tB, K):
    """M, N over the 64-wide tile edges, (alpha, beta) cycling over all nine pairs; the products the planner sends to the tensor
    cores (NT, alpha = 1, beta in {0, 1}, K = 100) are only checked to do so here -- the integer suite below covers them"""
    k = 0
    for M in MNS:
        for N in MNS:
            alpha, beta = ALPHA_BETA[(k + K) % len(ALPHA_BETA)]
            k += 1
            sa, sb = op_shapes(tA, tB, M, N, K)
            a = rng.standard_normal(sa).astype(np.float32)
            b = rng.standard_normal(sb).astype(np.float32)
            c0 = rng.standard_normal((M, N)).astype(np.float32)
            g = Gemm(tA, tB, M, N, K, alpha, beta, a, b)
            q = g.plan()
            if goes_tc(tA, tB, K, alpha, beta):
                assert q["route"] == "tc", (M, N, K, alpha, beta, q)
                continue
            assert q == ffma_plan(M, N, K), (M, N, K, alpha, beta, q)
            got = check_ffma(g, a, b, c0)
            if K == 0:                                  # no products: alpha * (+0) + beta * C
                assert np.array_equal(got, np.float32(beta) * c0) if beta else not got.any()


# ---- GEMV: bit-exact --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("beta", [0.0, 1.0])
@pytest.mark.parametrize("tA", [0, 1], ids=["N", "T"])
def test_gemv_bit_exact(rng, tA, beta):
    for M in (1, 7, 129, 3000):
        for N in (1, 31, 32, 33, 1000):
            alpha = -3.0 if (M + N) % 2 else 1.0
            A = rng.standard_normal((M, N)).astype(np.float32)
            x = rng.standard_normal(M if tA else N).astype(np.float32)
            ny = N if tA else M
            y0 = rng.standard_normal(ny).astype(np.float32)
            buf = torch.full((GUARD + ny + GUARD,), float(SENTINEL), device="cuda")
            buf[GUARD:GUARD + ny] = float("nan") if beta == 0.0 else dev(y0)
            capi.sgemv(tA, M, N, alpha, dev(A), dev(x), beta, buf[GUARD:GUARD + ny])
            out = host(buf)
            assert (bits(np.concatenate([out[:GUARD], out[GUARD + ny:]])) == bits(SENTINEL)).all(), "write outside y"
            got = out[GUARD:GUARD + ny]
            ok = o.ffma_match(got, o.gemv_ffma(tA, M, N, alpha, A, x, beta, y0))
            assert ok.all(), (M, N, alpha, f"{(~ok).sum()} elements differ, first at {np.argwhere(~ok)[0]}")


# ---- tensor-core NT route, integer data: equal to the float64 product --------------------------------------------------------
def nkb(K):
    return (K + 63) // 64


# (id, (M, N, K, workspace, beta, c_off) as a function of the SM count, regime the plan must show)
TC_INT = [
    ("cols64_splits", lambda S: (128, 64, 64 * 40, "planned", 0.0, 0),
     lambda q, S: q["cols"] == 64 and q["splits"] > 1),
    ("cols128_beta1", lambda S: (128, 128, 64 * 40, "planned", 1.0, 0),
     lambda q, S: q["cols"] == 128 and q["splits"] > 1),
    ("m1", lambda S: (1, 64, 64 * 12 + 4, "planned", 1.0, 0),
     lambda q, S: q["m_tiles"] == 1 and q["splits"] > 1 and q["bpi"] == 13),
    ("m127", lambda S: (127, 100, 64 * 12 + 60, "planned", 0.0, 0),
     lambda q, S: q["m_tiles"] == 1 and q["cols"] == 128),
    ("m129", lambda S: (129, 96, 256, None, 1.0, 0),
     lambda q, S: q["m_tiles"] == 2 and q["splits"] == 1),
    ("n1", lambda S: (200, 1, 68, "planned", 0.0, 0),
     lambda q, S: q["cols"] == 64 and q["n_tiles"] == 1 and q["bpi"] == 2),
    ("n63", lambda S: (64, 63, 124, None, 1.0, 0),
     lambda q, S: q["cols"] == 64 and q["splits"] == 1 and q["bpi"] == 2),
    ("n65_k64", lambda S: (64, 65, 64, "planned", 0.0, 0),
     lambda q, S: q["cols"] == 128 and q["bpi"] == 1 and q["splits"] == 1),
    ("n129", lambda S: (256, 129, 64 * 9 + 4, "planned", 1.0, 0),
     lambda q, S: q["cols"] == 128 and q["n_tiles"] == 2 and q["m_tiles"] == 2 and q["splits"] > 1),
    ("one_split_no_workspace", lambda S: (300, 200, 64 * 30 + 60, None, 0.0, 0),
     lambda q, S: q["splits"] == 1 and q["kb_per_split"] == q["bpi"] == 31),
    ("one_split_tiles_ge_sms", lambda S: (128 * 12, 128 * -(-S // 12), 64 * 9, "planned", 1.0, 0),
     lambda q, S: q["splits"] == 1 and q["m_tiles"] * q["n_tiles"] >= S),
    ("splits_ragged", lambda S: (256, 128, 64 * (S // 2 * 3 + 1), "planned", 0.0, 0),
     lambda q, S: q["splits"] > 1 and q["bpi"] % q["kb_per_split"] != 0),
    ("splits_near_sms", lambda S: (96, 40, 64 * (5 * S - 3), "planned", 1.0, 0),
     lambda q, S: q["splits"] >= 0.9 * S and q["bpi"] % q["kb_per_split"] != 0),
    ("c_offset_splits", lambda S: (129, 65, 64 * 20 + 4, "planned", 1.0, 1),
     lambda q, S: q["splits"] > 1),
    ("c_offset_one_split", lambda S: (65, 129, 64 * 3 + 60, None, 0.0, 1),
     lambda q, S: q["splits"] == 1),
]


def small_ints(rng, shape, lim=8):
    return rng.integers(-lim, lim + 1, shape).astype(np.float32)


@pytest.mark.parametrize("cid,shape,regime", TC_INT, ids=[c[0] for c in TC_INT])
def test_tc_integer_exact(rng, sms, cid, shape, regime):
    M, N, K, ws, beta, c_off = shape(sms)
    a, b = small_ints(rng, (M, K)), small_ints(rng, (N, K))
    c0 = small_ints(rng, (M, N), 1000)
    g = Gemm(0, 1, M, N, K, 1.0, beta, a, b, ws=ws, c_off=c_off)
    q = g.plan()
    assert q["route"] == "tc" and q["bpi"] == nkb(K), q
    assert regime(q, sms), f"{cid}: the planner no longer produces this case's regime; plan {q}"
    want = (a.astype(np.float64) @ b.astype(np.float64).T + (c0 if beta else 0.0)).astype(np.float32)
    got = g.checked(c0)
    bad = np.argwhere(bits(got) != bits(want))
    assert bad.size == 0, f"{len(bad)} elements differ, first at {tuple(bad[0])}: got {got[tuple(bad[0])]}, want {want[tuple(bad[0])]}"


@pytest.mark.parametrize("ws", ["short", "misaligned"])
def test_tc_workspace_fallback_is_one_split(rng, ws):
    """a workspace too short by 4 bytes, or at a 4-byte offset: the tensor-core route with one split, the bits of b2c_sgemm"""
    M, N, K = 128, 128, 64 * 40
    a, b = small_ints(rng, (M, K)), rng.standard_normal((N, K)).astype(np.float32)
    c0 = rng.standard_normal((M, N)).astype(np.float32)
    planned = Gemm(0, 1, M, N, K, 1.0, 1.0, a, b).plan()
    assert planned["splits"] > 1, planned
    g = Gemm(0, 1, M, N, K, 1.0, 1.0, a, b, ws=ws)
    q = g.plan()
    assert q["route"] == "tc" and q["splits"] == 1 and q["kb_per_split"] == q["bpi"], q
    plain = Gemm(0, 1, M, N, K, 1.0, 1.0, a, b, ws=None)
    assert plain.plan() == q
    assert np.array_equal(bits(g.checked(c0)), bits(plain.call(c0)))


# ---- tensor-core NT route, float data: the per-element bound -------------------------------------------------------------------
def scaled(rng, rows, cols, period):
    """N(0, 1) rows scaled by 2^-(row % period): sum |ab| spans decades across the output"""
    return (rng.standard_normal((rows, cols)) * np.exp2(-(np.arange(rows) % period))[:, None]).astype(np.float32)


def tc_bound(q, mag, ref):
    n = 12 * q["kb_per_split"] + q["splits"] + 1
    return (2.0 ** -16 + n * 2.0 ** -23) * mag + 2.0 ** -24 * np.abs(ref)


def check_float(g, a, b, c0, label):
    q = g.plan()
    got = g.checked(c0)
    a64, b64 = a.astype(np.float64), b.astype(np.float64)
    ref = a64 @ b64.T + (c0 if g.beta else 0.0)
    mag = np.abs(a64) @ np.abs(b64).T
    err = np.abs(got - ref)
    blob = rel_err(got, ref)
    if q["route"] == "ffma":
        bound = o.gemm_ffma(0, 1, g.M, g.N, g.K, 1.0, a, b, g.beta, c0 if g.beta else np.zeros((g.M, g.N), np.float32))
        ok = o.ffma_match(got, bound)
        print(f"[gemm] {label}: plan {q}; FFMA chain bit-exact on {ok.mean():.6f} of the elements; blob err {blob:.3g}, "
              f"max err / sum|ab| {np.max(err / mag):.3g}")
        assert ok.all()
    else:
        bnd = tc_bound(q, mag, ref)
        print(f"[gemm] {label}: plan {q}; blob err {blob:.3g}; max err / sum|ab| {np.max(err / mag):.3g}; "
              f"max err / bound {np.max(err / bnd):.3g}")
        bad = np.argwhere(err > bnd)
        assert bad.size == 0, f"{len(bad)} elements over the bound, first at {tuple(bad[0])}"
    assert blob < TOL, blob
    return q


# InnerProduct forward at models.BASELINE_BATCH: (id, net, M, N, K)
IP_FC = [("alexnet_fc6", "alexnet", 4096, 9216), ("alexnet_fc7", "alexnet", 4096, 4096), ("alexnet_fc8", "alexnet", 1000, 4096),
         ("vgg16_fc6", "vgg16", 4096, 25088), ("resnet50_fc1000", "resnet50", 1000, 2048), ("googlenet_loss3", "googlenet", 1000, 1024)]


@pytest.mark.parametrize("ws", ["planned", None], ids=["sgemm_ex", "sgemm"])
@pytest.mark.parametrize("cid,net,N,K", IP_FC, ids=[c[0] for c in IP_FC])
def test_tc_inner_product_shapes(rng, cid, net, N, K, ws):
    M = models.BASELINE_BATCH[net]
    x = np.maximum(scaled(rng, M, K, 7), 0)            # post-ReLU activations
    w = scaled(rng, N, K, 9) * np.float32(0.02)
    g = Gemm(0, 1, M, N, K, 1.0, 0.0, x, w, ws=ws)
    q = g.plan()
    # without its workspace a product the planner splits runs unsplit, and past 256 K blocks on the FFMA kernel (VGG-16 fc6)
    assert q["route"] == ("tc" if ws is not None or nkb(K) <= 256 else "ffma"), q
    check_float(g, x, w, None, f"{cid} M={M} N={N} K={K} {'with' if ws else 'without'} workspace")


def test_long_unsplit_chain(rng):
    """NT, M = 64, N = 27, K = 50176 without a workspace: what the CAFFE engine's per-image weight gradient of VGG-16 conv1 asks for.
    Unsplit on the tensor cores its one accumulator chain of 784 K blocks measured 1.9e-4 against the 1e-4 bar; it runs on the FFMA
    kernel, and the limit sits at 256 blocks"""
    M, N, K = 64, 27, 50176
    for kb, route in ((256, "tc"), (257, "ffma")):
        assert capi.sgemm_plan(0, 1, M, N, 64 * kb, 1.0, 1.0, 256, 256)["route"] == route, kb
        with_ws = capi.sgemm_plan(0, 1, M, N, 64 * kb, 1.0, 1.0, 256, 256, 256, capi.lib().b2c_sgemm_workspace_bytes(0, 1, M, N, 64 * kb))
        assert with_ws["route"] == "tc" and with_ws["splits"] > 1, with_ws
    dy = scaled(rng, M, K, 6)
    col = scaled(rng, N, K, 5)
    g = Gemm(0, 1, M, N, K, 1.0, 1.0, dy, col, ws=None)
    assert g.plan() == ffma_plan(M, N, K), g.plan()
    c0 = rng.standard_normal((M, N)).astype(np.float32)
    check_float(g, dy, col, c0, "long unsplit chain M=64 N=27 K=50176")


# ---- fallbacks to the FFMA kernel: by plan and by bits -------------------------------------------------------------------------
@pytest.fixture
def default_math_algo():
    """b2c_set_default_math / _algo are process-wide: put them back whatever the test does"""
    yield capi.lib()
    L = capi.lib()
    capi.check(L.b2c_set_default_math(capi.MATH_FP32))
    capi.check(L.b2c_set_default_algo(capi.ALGO_AUTO))


FALLBACKS = [  # (id, M, N, K, alpha, beta, a_off, b_off, math, algo)
    ("a_offset_4", 130, 70, 256, 1.0, 0.0, 1, 0, None, None),
    ("b_offset_4", 130, 70, 256, 1.0, 1.0, 0, 1, None, None),
    ("alpha_0_5", 130, 70, 256, 0.5, 1.0, 0, 0, None, None),
    ("beta_minus_2", 130, 70, 256, 1.0, -2.0, 0, 0, None, None),
    ("k_lt_64", 130, 70, 60, 1.0, 0.0, 0, 0, None, None),
    ("k_mod4_2", 130, 70, 258, 1.0, 1.0, 0, 0, None, None),
    ("tf32_default_math", 130, 70, 256, 1.0, 0.0, 0, 0, capi.MATH_TF32, None),
    ("simt_default_algo", 130, 70, 256, 1.0, 1.0, 0, 0, None, capi.ALGO_SIMT),
]


@pytest.mark.parametrize("cid,M,N,K,alpha,beta,a_off,b_off,math,algo", FALLBACKS, ids=[c[0] for c in FALLBACKS])
def test_nt_fallback_to_ffma(rng, default_math_algo, cid, M, N, K, alpha, beta, a_off, b_off, math, algo):
    L = default_math_algo
    if math is not None:
        capi.check(L.b2c_set_default_math(math))
    if algo is not None:
        capi.check(L.b2c_set_default_algo(algo))
    a = rng.standard_normal((M, K)).astype(np.float32)
    b = rng.standard_normal((N, K)).astype(np.float32)
    c0 = rng.standard_normal((M, N)).astype(np.float32)
    g = Gemm(0, 1, M, N, K, alpha, beta, a, b, a_off=a_off, b_off=b_off)
    assert g.plan() == ffma_plan(M, N, K), g.plan()
    check_ffma(g, a, b, c0)


# ---- InnerProduct through TrainNet: forward, dW, db and dx -----------------------------------------------------------------------
SOLVER = 'base_lr: 0.01 lr_policy: "fixed" max_iter: 10 solver_mode: GPU'


def ip_net(M, K, N, aux):
    """Input -> InnerProduct (bias) -> EuclideanLoss, force_backward so dx is computed.  aux: a 2-weight InnerProduct on its own
    input ahead of it: its slot (2 floats) puts the checked layer's weight 8 bytes past a 16-byte boundary in the arena"""
    shapes = f"shape {{ dim: {M} dim: {K} }} shape {{ dim: {M} dim: {N} }}" + (f" shape {{ dim: {M} dim: 2 }}" if aux else "")
    tops = 'top: "data" top: "target"' + (' top: "aux"' if aux else "")
    txt = f'name: "ip"\nforce_backward: true\nlayer {{ name: "input" type: "Input" {tops} input_param {{ {shapes} }} }}\n'
    if aux:
        txt += ('layer { name: "ip_aux" type: "InnerProduct" bottom: "aux" top: "aux_out" '
                'inner_product_param { num_output: 1 bias_term: false } }\n')
    txt += (f'layer {{ name: "fc" type: "InnerProduct" bottom: "data" top: "fc" inner_product_param {{ num_output: {N} }} }}\n'
            'layer { name: "loss" type: "EuclideanLoss" bottom: "fc" bottom: "target" top: "loss" }\n')
    return txt


def run_ip(M, K, N, x, w, bias, target, bwd_tc, aux=False):
    """one forward_backward() with B2C_IP_BWD_TC at its default (bwd_tc) or 0; the switch stays set for the whole run, since
    InnerProductLayer::Reshape reads it whenever the net reshapes"""
    old = os.environ.get("B2C_IP_BWD_TC")
    if bwd_tc:
        os.environ.pop("B2C_IP_BWD_TC", None)
    else:
        os.environ["B2C_IP_BWD_TC"] = "0"
    try:
        t = host_api.Trainer(ip_net(M, K, N, aux), SOLVER, num_classes=N)
        layers = [nm for nm, _ in t.layers()]
        fc = layers.index("fc")
        p0 = 1 if aux else 0                             # ip_aux's weight comes first in the arena
        if aux:
            t.set_param(0, np.ones(2, np.float32))
            t.set_blob("aux", np.ones((M, 2), np.float32))
        t.set_param(p0, w)
        t.set_param(p0 + 1, bias)
        t.set_blob("data", x)
        t.set_blob("target", target)
        _, wptr, _ = t.layer_blob_pointers(fc, 0)
        before = capi.lib().b2c_launch_count()
        t.forward_backward()
        launches = capi.lib().b2c_launch_count() - before
        out = dict(y=t.get_blob("fc").reshape(M, N), dw=t.get_param(p0, 1).reshape(N, K), db=t.get_param(p0 + 1, 1),
                   dx=t.get_blob("data", diff=True).reshape(M, K), wptr=wptr, launches=launches)
        del t
    finally:
        if old is None:
            os.environ.pop("B2C_IP_BWD_TC", None)
        else:
            os.environ["B2C_IP_BWD_TC"] = old
    return out


def ip_integer_data(rng, M, K, N):
    x, w, bias = small_ints(rng, (M, K), 3), small_ints(rng, (N, K), 3), small_ints(rng, N, 50)
    y = x.astype(np.float64) @ w.astype(np.float64).T + bias
    d = rng.integers(-4, 5, (M, N)).astype(np.float64)
    return x, w, bias, (y - d).astype(np.float32), y, d


def assert_equal(got, want, what):
    want = np.asarray(want).astype(np.float32)
    bad = np.argwhere(bits(got) != bits(want))
    assert bad.size == 0, f"{what}: {len(bad)} elements differ, first at {tuple(bad[0])}: got {got[tuple(bad[0])]}, want {want[tuple(bad[0])]}"


@pytest.mark.parametrize("M,N,aux", [(512, 4096, False), (1024, 1024, False), (512, 1024, True)],
                         ids=["batch512", "batch1024", "batch512_w_8_byte_slot"])
def test_inner_product_exact(rng, M, N, aux):
    """integer x, W, b and targets y - d (d in [-4, 4]): dy = d / M is exact in bf16, so y, dW, db and dx equal float64 whichever
    kernels run -- the tensor-core backward (dW via two transposes and a split-K NT GEMM with beta = 1, batch >= 512) or the FFMA
    one (B2C_IP_BWD_TC=0)"""
    K = 9216
    assert capi.lib().b2c_sgemm_tc_supported(0, 1, N, K, M) == 1 and capi.lib().b2c_sgemm_tc_supported(0, 1, M, K, N) == 1
    x, w, bias, target, y, d = ip_integer_data(rng, M, K, N)
    dy = d / M
    want = dict(y=y, dw=dy.T @ x.astype(np.float64), db=dy.sum(0), dx=dy @ w.astype(np.float64))
    runs = {}
    for tc in (True, False):
        r = run_ip(M, K, N, x, w, bias, target, tc, aux)
        assert r["wptr"] % 16 == (8 if aux else 0), hex(r["wptr"])
        # the forward's operand: an 8-byte slot would send it to the FFMA kernel, so the layer copies W to an aligned buffer
        fwd = capi.sgemm_plan(0, 1, M, N, K, 1.0, 0.0, 256, r["wptr"])
        assert fwd["route"] == ("ffma" if aux else "tc"), fwd
        for k in want:
            assert_equal(r[k], want[k], f"{k} (B2C_IP_BWD_TC {'default' if tc else '0'})")
        runs[tc] = r
    # the tensor-core backward adds three transposes (dY and X for dW, W for dx) and replaces one FFMA launch by one tensor-core
    # launch for each of dW and dx; ip_aux (K = 2, batch >= 512) takes the tensor-core dW too: two more transposes
    extra = 3 + (2 if aux else 0)
    assert runs[True]["launches"] - runs[False]["launches"] == extra, (runs[True]["launches"], runs[False]["launches"])


def test_inner_product_batch_520(rng):
    """batch 520: 1/520 is not exact, and the dW GEMM's K (the batch) ends in an 8-wide tail; checked with the float bound"""
    M, K, N = 520, 9216, 1024
    x, w, bias, target, y, d = ip_integer_data(rng, M, K, N)
    r = run_ip(M, K, N, x, w, bias, target, True)
    assert_equal(r["y"], y, "y")
    alpha = np.float32(1.0) / np.float32(M)
    dy = (alpha * d.astype(np.float32)).astype(np.float64)      # b2c_euclidean_loss_backward: fl(alpha * diff)
    # the layer's backward workspace holds the larger of the two GEMMs' planned workspaces: both run their planned splits
    L = capi.lib()
    ws = max(L.b2c_sgemm_workspace_bytes(0, 1, N, K, M), L.b2c_sgemm_workspace_bytes(0, 1, M, K, N))
    q_dw = capi.sgemm_plan(0, 1, N, K, M, 1.0, 1.0, 256, 256, 256, ws)          # dW[N x K] += dY^T (x^T)^T, K = the batch
    q_dx = capi.sgemm_plan(0, 1, M, K, N, 1.0, 0.0, 256, 256, 256, ws)          # dx[M x K] = dY (W^T)^T
    assert q_dw["route"] == "tc" and q_dw["bpi"] == 9 and q_dx["route"] == "tc", (q_dw, q_dx)
    for name, q, got, ref, mag in (("dw", q_dw, r["dw"], dy.T @ x, np.abs(dy).T @ np.abs(x)),
                                   ("dx", q_dx, r["dx"], dy @ w, np.abs(dy) @ np.abs(w))):
        bnd = tc_bound(q, mag, ref)
        err = np.abs(got - ref)
        print(f"[gemm] InnerProduct batch 520 {name}: plan {q}; blob err {rel_err(got, ref):.3g}, "
              f"max err / bound {np.max(err / bnd):.3g}")
        assert (err <= bnd).all(), name
        assert rel_err(got, ref) < TOL
    # db: b2c_bias_backward's fp32 sum over the batch
    assert np.all(np.abs(r["db"] - dy.sum(0)) <= gamma_f32(M) * np.abs(dy).sum(0))


def gamma_f32(n):
    return n * 2.0 ** -24 / (1 - n * 2.0 ** -24)

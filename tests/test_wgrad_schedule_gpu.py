"""Schedule edge cases of the weight-gradient kernels against the float64 CPU oracle.

b2c_conv_backward_filter picks one of several kernels (include/b2c.h, b2c_wgrad_route): the TMA-staged bf16x3 kernel for
3x3 / pad 1 and 1x1 maps (8-channel x 9-tap tiles, or 64 / 128 channels; plane mode on 7x7 maps), the TMA-fed 3xTF32 1x1
kernel for small maps, compaction of strided 1x1 layers in front of either, and the gather kernel for everything else.  Each
splits the pixel reduction over one wave of CTAs and adds the partial tiles in split order.  Every case below states the
schedule regime it exists for as an assertion on ConvDesc.wgrad_plan() (b2c_debug_wgrad_plan, the planner the launch runs),
so a planner change that moves a case off its path fails here, naming the regime, instead of silently testing something else.
Shapes are chosen for 132 SMs and scaled by the device's SM count where the plan depends on it.

Every case runs through the C ABI with a workspace full of NaN (a split-K partial read before it is written shows up) and dW
as a view inside a buffer whose head and tail hold a sentinel (a write outside dW shows up), on top of a random dW0 the
gradient must be added to:
  * parity with the oracle at the 1e-4 blob-level bar, and no NaN;
  * a second call is bit-identical (the workspace then holds the first call's leftovers instead of NaN);
  * dY = 0 leaves dW bit-identical to dW0 (stale accumulators or partials would not).
The staged and gather routes also get impulse tests, which check every element: dY (or X) is zero except a few entries, one per
output channel (or input channel), placed at image corners, row ends, the last image and the first pixel of the K block a split
boundary falls in.  Then each dW element either stays bit-identical to dW0 or equals dW0 + one product, to within the bf16x3 /
3xTF32 error of that product.  A wrong tap mask or row wrap moves a few border terms, which a blob-level bar cannot see."""
import ctypes as C

import numpy as np
import pytest

import oracle as o
from cases import make, rel_err

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import caffe_mpi_b200 as m  # noqa: E402
from caffe_mpi_b200 import capi  # noqa: E402

TOL = 1e-4
GUARD = 64                                   # sentinel floats before and after dW (256 bytes: dW stays 16-byte aligned)
SENTINEL = np.float32(-7.25e19)
STAGED = ("staged_3x3", "staged_3x3_plane", "staged_1x1", "staged_1x1_plane")


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


def conv(N, C, H, W, O, k, s=1, p=None, d=1, G=1):
    kk = k if isinstance(k, int) else k[0]
    return dict(N=N, Cin=C, H=H, W=W, O=O, k=k, s=s, p=(kk // 2 if p is None else p), d=d, G=G, bias=False)


def last_split_len(q):
    return q["nkb"] - (q["splits"] - 1) * q["per"]


def mid_image_splits(q):
    """some split starts inside an image (the K blocks of an image are divided between two CTAs)"""
    return q["bpi"] > 0 and q["splits"] > 1 and q["per"] % q["bpi"] != 0


# (id, shape as a function of the SM count, regime the plan must show, math mode, impulse tests)
# The regime is a predicate over the plan dict {route, splits, per, nkb, cols, bpi} and the SM count.
CASES = [
    # ---- staged 3x3 (wgrad_stg_kernel<9, 8, false>): 64-pixel K blocks, accumulator folded into `tot` every 8 blocks
    ("s3_115_splits_mid_image", lambda S: conv(200 * S // 132, 8, 16, 16, 32, 3),
     lambda q, S: q["route"] == "staged_3x3" and q["splits"] >= 9 and q["splits"] % 8 != 0 and q["nkb"] % q["per"] != 0
     and mid_image_splits(q), None, True),
    ("s3_splits_near_sm_count", lambda S: conv(130 * S // 132, 8, 16, 16, 32, 3),
     lambda q, S: q["route"] == "staged_3x3" and q["splits"] > 0.9 * S and q["splits"] % 8 != 0, None, False),
    ("s3_promote_per9", lambda S: conv(27, 8 * (S // 3), 8, 8, 128, 3),
     lambda q, S: q["route"] == "staged_3x3" and q["per"] == 9 and q["splits"] > 1 and q["nkb"] % 9 == 0, None, True),
    ("s3_promote_last_split_8", lambda S: conv(26, 8 * (S // 3), 8, 8, 128, 3),
     lambda q, S: q["route"] == "staged_3x3" and q["per"] == 9 and last_split_len(q) == 8, None, False),
    ("s3_one_split", lambda S: conv(3, 8 * (S + 1), 8, 8, 32, 3),
     lambda q, S: q["route"] == "staged_3x3" and q["splits"] == 1 and q["nkb"] == 3, None, True),
    ("s3_1x64_one_x_stage", lambda S: conv(40, 16, 1, 64, 32, 3),
     lambda q, S: q["route"] == "staged_3x3" and q["bpi"] == 1 and q["splits"] > 1, None, True),
    ("s3_64x1", lambda S: conv(40, 16, 64, 1, 32, 3),
     lambda q, S: q["route"] == "staged_3x3" and q["bpi"] == 1 and q["splits"] > 1, None, True),
    ("s3_32x2", lambda S: conv(12, 8, 32, 2, 24, 3), lambda q, S: q["route"] == "staged_3x3", None, True),
    ("s3_24x3", lambda S: conv(12, 8, 24, 3, 24, 3), lambda q, S: q["route"] == "staged_3x3" and q["bpi"] == 2, None, True),
    ("s3_3x32", lambda S: conv(9, 8, 3, 32, 32, 3),
     lambda q, S: q["route"] == "staged_3x3" and q["bpi"] == 2 and mid_image_splits(q), None, True),
    ("s3_4x17_padding_block", lambda S: conv(9, 8, 4, 17, 32, 3),
     lambda q, S: q["route"] == "staged_3x3" and q["bpi"] == 2 and mid_image_splits(q), None, True),
    ("s3_c12_o136", lambda S: conv(6, 12, 12, 12, 136, 3), lambda q, S: q["route"] == "staged_3x3" and q["splits"] > 1,
     None, True),
    ("s3_c20_o24", lambda S: conv(6, 20, 12, 12, 24, 3), lambda q, S: q["route"] == "staged_3x3" and q["splits"] > 1,
     None, True),
    ("s3_c24_o40", lambda S: conv(6, 24, 12, 12, 40, 3), lambda q, S: q["route"] == "staged_3x3" and q["splits"] > 1,
     None, True),
    ("s3_w90_one_x_stage_18_splits", lambda S: conv(6, 8, 8, 90, 32, 3),
     lambda q, S: q["route"] == "staged_3x3" and q["splits"] == 18 and mid_image_splits(q), None, True),
    # ---- staged plane mode (7x7 maps, one image per K block)
    ("p3_c12_o20", lambda S: conv(64, 12, 7, 7, 20, 3),
     lambda q, S: q["route"] == "staged_3x3_plane" and q["splits"] > 1 and q["bpi"] == 1, None, True),
    ("p1_c4_o4", lambda S: conv(70, 4, 7, 7, 4, 1),
     lambda q, S: q["route"] == "staged_1x1_plane" and q["splits"] > 1 and q["cols"] == 64, None, True),
    ("p1_c200_o132", lambda S: conv(40, 200, 7, 7, 132, 1),
     lambda q, S: q["route"] == "staged_1x1_plane" and q["cols"] == 128 and q["splits"] > 1, None, True),
    ("p3_c10_gather", lambda S: conv(16, 10, 7, 7, 20, 3), lambda q, S: q["route"] == "gather", None, True),
    # ---- staged 1x1 (wgrad_stg_kernel<1, 64 / 128, false>)
    ("s1_c3_o129", lambda S: conv(10, 3, 8, 8, 129, 1), lambda q, S: q["route"] == "staged_1x1" and q["cols"] == 64, None, True),
    ("s1_c64_o1", lambda S: conv(10, 64, 8, 8, 1, 1), lambda q, S: q["route"] == "staged_1x1" and q["cols"] == 64, None, True),
    ("s1_c65_o127", lambda S: conv(10, 65, 8, 8, 127, 1), lambda q, S: q["route"] == "staged_1x1" and q["cols"] == 128,
     None, True),
    ("s1_c200_o129", lambda S: conv(10, 200, 8, 8, 129, 1), lambda q, S: q["route"] == "staged_1x1" and q["cols"] == 128,
     None, True),
    ("s1_75_splits", lambda S: conv(300 * S // 132, 32, 8, 8, 32, 1),
     lambda q, S: q["route"] == "staged_1x1" and q["splits"] >= 9 and q["splits"] % 8 != 0, None, True),
    ("s1_6x12_mid_image", lambda S: conv(9, 64, 6, 12, 64, 1),
     lambda q, S: q["route"] == "staged_1x1" and q["bpi"] == 2 and mid_image_splits(q), None, True),
    # ---- TMA-fed 1x1 (wgrad1x1_tma_kernel<32 / 64 / 128>): 32 <= H*W < 64
    ("t1_6x6_nt32", lambda S: conv(40, 20, 6, 6, 64, 1),
     lambda q, S: q["route"] == "tma_1x1" and q["cols"] == 32 and q["splits"] >= 9, None, False),
    ("t1_4x8_nt64", lambda S: conv(80, 48, 4, 8, 64, 1),
     lambda q, S: q["route"] == "tma_1x1" and q["cols"] == 64 and q["splits"] >= 9, None, False),
    ("t1_6x10_nt128", lambda S: conv(40, 200, 6, 10, 64, 1),
     lambda q, S: q["route"] == "tma_1x1" and q["cols"] == 128 and q["splits"] >= 9, None, False),
    # ---- compaction of strided 1x1 layers
    ("c_14_to_7_plane", lambda S: conv(20, 64, 14, 14, 40, 1, s=2), lambda q, S: q["route"] == "compact_staged" and q["bpi"] == 1,
     None, False),
    ("c_13_to_7_plane", lambda S: conv(20, 64, 13, 13, 40, 1, s=2), lambda q, S: q["route"] == "compact_staged" and q["bpi"] == 1,
     None, False),
    ("c_16_to_8", lambda S: conv(20, 64, 16, 16, 40, 1, s=2), lambda q, S: q["route"] == "compact_staged" and q["bpi"] == 1,
     None, False),
    ("c_12_to_6_tma", lambda S: conv(20, 32, 12, 12, 136, 1, s=2), lambda q, S: q["route"] == "compact_tma", None, False),
    ("c_12_to_6_o96_gather", lambda S: conv(20, 32, 12, 12, 96, 1, s=2), lambda q, S: q["route"] == "gather", None, False),
    ("c_stride_2x1", lambda S: conv(12, 32, 16, 8, 40, 1, s=(2, 1)), lambda q, S: q["route"] == "compact_staged", None, False),
    ("c_stride_1x2", lambda S: conv(12, 32, 8, 16, 40, 1, s=(1, 2)), lambda q, S: q["route"] == "compact_staged", None, False),
    ("c_stride_3", lambda S: conv(12, 32, 24, 24, 40, 1, s=3), lambda q, S: q["route"] == "compact_staged", None, False),
    # ---- gather kernel (igemm_wgrad_kernel<32 / 64, SPLIT, X1X1>): 32-pixel K blocks over the flattened pixels, promoted
    # into shared memory every 16 blocks
    ("g_5x5_p2", lambda S: conv(4, 16, 12, 12, 32, 5), lambda q, S: q["route"] == "gather" and q["cols"] == 64, None, True),
    ("g_stem_7x7_s2", lambda S: conv(4, 3, 56, 56, 64, 7, s=2, p=3),
     lambda q, S: q["route"] == "gather" and q["cols"] == 64 and q["splits"] > 1, None, True),
    ("g_group2", lambda S: conv(4, 16, 10, 10, 32, 3, G=2), lambda q, S: q["route"] == "gather" and q["cols"] == 64, None, True),
    ("g_dilation2", lambda S: conv(4, 16, 12, 12, 32, 3, p=2, d=2), lambda q, S: q["route"] == "gather", None, True),
    ("g_13x13_per_ge17", lambda S: conv(24, 64, 13, 13, 256, 3),
     lambda q, S: q["route"] == "gather" and q["per"] >= 17 and q["splits"] > 1, None, True),
    ("g_1x1_4x4", lambda S: conv(24, 16, 4, 4, 40, 1), lambda q, S: q["route"] == "gather" and q["cols"] == 32, None, True),
    ("g_1x1_5x5", lambda S: conv(24, 48, 5, 5, 40, 1), lambda q, S: q["route"] == "gather" and q["cols"] == 64, None, True),
    ("g_kd27_nt32", lambda S: conv(8, 3, 13, 13, 16, 3),
     lambda q, S: q["route"] == "gather" and q["cols"] == 32 and q["splits"] > 1, None, True),
    # single-pass TF32: the gather kernel's non-SPLIT instantiation (1e-3 bar)
    ("g_tf32", lambda S: conv(8, 16, 16, 16, 32, 3), lambda q, S: q["route"] == "gather", capi.MATH_TF32, False),
]
IDS = [c[0] for c in CASES]


class Run:
    """One descriptor and its inputs; calls b2c_conv_backward_filter through the C ABI with a NaN-filled workspace and dW
    inside a sentinel-guarded buffer."""

    def __init__(self, c, math=None):
        self.c, self.po, self.pc = c, make(o, c), make(capi, c)
        self.d = m.ConvDesc(self.pc, math=math)
        self.n = int(np.prod(self.po.w_shape()))

    def plan(self):
        return self.d.wgrad_plan()

    def call(self, x, dy, dw0, x_off=0, dy_off=0, ws_fill=0xFF):
        """dW0 + gradient; checks the guard bands.  x_off / dy_off: element offset of the operand inside its buffer."""
        need = self.d.workspace_bytes(capi.OP_BACKWARD_FILTER)
        ws = torch.full((max(need, 16),), ws_fill, dtype=torch.uint8, device="cuda")
        buf = torch.full((GUARD + self.n + GUARD,), float(SENTINEL), device="cuda")
        buf[GUARD:GUARD + self.n] = dev(dw0.reshape(-1))
        X = torch.empty(x.size + x_off, device="cuda")
        X[x_off:] = dev(x.reshape(-1))
        DY = torch.empty(dy.size + dy_off, device="cuda")
        DY[dy_off:] = dev(dy.reshape(-1))
        L = capi.lib()
        capi.check(L.b2c_conv_backward_filter(self.d._h, C.c_void_p(X[x_off:].data_ptr()), C.c_void_p(DY[dy_off:].data_ptr()),
                                              C.c_void_p(buf[GUARD:].data_ptr()), C.c_void_p(ws.data_ptr()), need,
                                              capi._stream()))
        out = host(buf)
        guard = np.concatenate([out[:GUARD], out[GUARD + self.n:]])
        assert (guard.view(np.int32) == SENTINEL.view(np.int32)).all(), "write outside dW"
        return out[GUARD:GUARD + self.n].reshape(self.po.w_shape())


def check_case(c, math, rng, tol):
    r = Run(c, math)
    x = rng.standard_normal(r.po.x_shape()).astype(np.float32)
    dy = rng.standard_normal(r.po.y_shape()).astype(np.float32)
    dw0 = rng.standard_normal(r.po.w_shape()).astype(np.float32)
    want, _, _ = o.conv_backward(r.po, x, np.zeros(r.po.w_shape(), np.float32), dy, dw=dw0, want_dx=False, acc64=True)
    got = r.call(x, dy, dw0)
    assert not np.isnan(got).any(), "NaN in dW: a split-K partial was read from the workspace before it was written"
    err = rel_err(got, want)
    assert err < tol, err
    again = r.call(x, dy, dw0, ws_fill=0x5A)
    assert np.array_equal(got.view(np.int32), again.view(np.int32)), "not bit-identical run to run"
    zero = r.call(x, np.zeros_like(dy), dw0)
    assert np.array_equal(zero.view(np.int32), dw0.view(np.int32)), "dY = 0 changed dW"
    return r


@pytest.mark.parametrize("cid,shape,regime,math,impulse", CASES, ids=IDS)
def test_wgrad_case(rng, sms, cid, shape, regime, math, impulse):
    c = shape(sms)
    q = Run(c, math).plan()
    assert regime(q, sms), f"{cid}: the planner no longer produces this case's regime; plan {q}"
    check_case(c, math, rng, 1e-3 if math == capi.MATH_TF32 else TOL)


# ---- impulse tests ----------------------------------------------------------------------------------------------------
def k_block_px(q):
    """pixels per K block: 64 on the staged kernel, 32 on the gather kernel"""
    return 64 if q["route"] in STAGED else 32


def positions(r, q, Hs, Ws):
    """(n, h, w) on an Hs x Ws map: corners, both ends of a middle row, the last image, and the first pixel of the K block
    the second and the last split start in"""
    N = r.po.N
    pts = [(0, 0, 0), (N - 1, 0, Ws - 1), (0, Hs - 1, 0), (N - 1, Hs - 1, Ws - 1), (N // 2, Hs // 2, 0),
           (N // 2, Hs // 2, Ws - 1), (0, Hs - 1, Ws - 1)]
    P = r.po.Ho * r.po.Wo
    for s in sorted({1, q["splits"] - 1}):
        if q["splits"] < 2 or s < 1:
            continue
        kb = s * q["per"]
        if q["bpi"]:                                  # staged: K blocks per image
            n, px = kb // q["bpi"], (kb % q["bpi"]) * k_block_px(q)
        else:                                         # gather: K blocks over the flattened (n, pixel) axis
            n, px = divmod(kb * 32, P)
        px = px * (Hs * Ws) // P                      # the same place on an input-sized map (dual test)
        pts.append((n, px // Ws, px % Ws))
    return list(dict.fromkeys(pts))


def expect_dy_impulses(po, x, dw0, imps):
    """dW0 + dY-impulse terms in float64, the per-element |product|, and the mask of elements that receive one"""
    exp = dw0.astype(np.float64).copy()
    mag = np.zeros_like(exp)
    hit = np.zeros(exp.shape, bool)
    Cg, Og = po.C // po.G, po.O // po.G
    for n, oc, ho, wo, v in imps:
        g = oc // Og
        for i in range(po.kh):
            for j in range(po.kw):
                ih, iw = ho * po.sh - po.ph + i * po.dh, wo * po.sw - po.pw + j * po.dw
                if 0 <= ih < po.H and 0 <= iw < po.W:
                    t = float(v) * x[n, g * Cg:(g + 1) * Cg, ih, iw].astype(np.float64)
                    exp[oc, :, i, j] += t
                    mag[oc, :, i, j] += np.abs(t)
                    hit[oc, :, i, j] = True
    return exp, mag, hit


def expect_x_impulses(po, dy, dw0, imps):
    exp = dw0.astype(np.float64).copy()
    mag = np.zeros_like(exp)
    hit = np.zeros(exp.shape, bool)
    Cg, Og = po.C // po.G, po.O // po.G
    for n, ch, ih, iw, v in imps:
        g, cl = ch // Cg, ch % Cg
        for i in range(po.kh):
            for j in range(po.kw):
                hh, ww = ih + po.ph - i * po.dh, iw + po.pw - j * po.dw
                if hh % po.sh or ww % po.sw:
                    continue
                ho, wo = hh // po.sh, ww // po.sw
                if 0 <= ho < po.Ho and 0 <= wo < po.Wo:
                    t = float(v) * dy[n, g * Og:(g + 1) * Og, ho, wo].astype(np.float64)
                    exp[g * Og:(g + 1) * Og, cl, i, j] += t
                    mag[g * Og:(g + 1) * Og, cl, i, j] += np.abs(t)
                    hit[g * Og:(g + 1) * Og, cl, i, j] = True
    return exp, mag, hit


def check_impulse_result(got, dw0, exp, mag, hit, what):
    miss = ~hit
    bad = np.argwhere(miss & (got.view(np.int32) != dw0.view(np.int32)))
    assert bad.size == 0, f"{what}: elements without a term changed, first at (o, c, i, j) = {tuple(bad[0])}"
    # bf16x3 / 3xTF32 keep a product to ~2^-16 relative; then one rounding of the add to dW0
    tol = 2.0 ** -14 * mag + 2.0 ** -22 * np.abs(exp) + 1e-30
    err = np.abs(got.astype(np.float64) - exp)
    bad = np.argwhere(hit & (err > tol))
    assert bad.size == 0, f"{what}: wrong term at (o, c, i, j) = {tuple(bad[0])}: got {got[tuple(bad[0])]}, want {exp[tuple(bad[0])]}"


@pytest.mark.parametrize("cid,shape,regime,math,impulse", [c for c in CASES if c[4]], ids=[c[0] for c in CASES if c[4]])
def test_wgrad_impulses(rng, sms, cid, shape, regime, math, impulse):
    r = Run(shape(sms), math)
    q = r.plan()
    assert q["route"] in STAGED + ("gather",), q
    po = r.po
    x = rng.standard_normal(po.x_shape()).astype(np.float32)
    dy = rng.standard_normal(po.y_shape()).astype(np.float32)
    dw0 = rng.standard_normal(po.w_shape()).astype(np.float32)
    # dY impulses: one per output channel, so every dW row holds at most one term per element
    pts = positions(r, q, po.Ho, po.Wo)
    for k0 in range(0, len(pts), po.O):
        chunk = pts[k0:k0 + po.O]
        chans = rng.permutation(po.O)[:len(chunk)]
        imps = [(n, int(oc), h, w, np.float32(rng.choice([-1, 1]) * rng.uniform(0.5, 2.0))) for (n, h, w), oc in zip(chunk, chans)]
        d1 = np.zeros_like(dy)
        for n, oc, h, w, v in imps:
            d1[n, oc, h, w] = v
        got = r.call(x, d1, dw0)
        check_impulse_result(got, dw0, *expect_dy_impulses(po, x, dw0, imps), f"dY impulses {imps}")
    # the dual: X impulses, one per input channel
    pts = positions(r, q, po.H, po.W)
    for k0 in range(0, len(pts), po.C):
        chunk = pts[k0:k0 + po.C]
        chans = rng.permutation(po.C)[:len(chunk)]
        imps = [(n, int(ch), h, w, np.float32(rng.choice([-1, 1]) * rng.uniform(0.5, 2.0))) for (n, h, w), ch in zip(chunk, chans)]
        x1 = np.zeros_like(x)
        for n, ch, h, w, v in imps:
            x1[n, ch, h, w] = v
        got = r.call(x1, dy, dw0)
        check_impulse_result(got, dw0, *expect_x_impulses(po, dy, dw0, imps), f"X impulses {imps}")


# ---- operands that are not 16-byte aligned: the gather kernel instead of the staged / TMA-fed one -------------------------
@pytest.mark.parametrize("operand", ["x", "dy"])
@pytest.mark.parametrize("cid,c,route", [("staged_3x3", conv(6, 16, 12, 12, 40, 3), "staged_3x3"),
                                         ("tma_1x1", conv(20, 48, 6, 6, 64, 1), "tma_1x1"),
                                         ("compact", conv(8, 32, 16, 16, 40, 1, s=2), "compact_staged")],
                         ids=["staged_3x3", "tma_1x1", "compact"])
def test_unaligned_operands_fall_back(rng, cid, c, route, operand):
    """a 4-byte offset on x or dy: the same answer within the bar, with exactly the workspace b2c_conv_workspace_bytes asks for"""
    r = Run(c)
    assert r.plan()["route"] == route
    po = r.po
    x = rng.standard_normal(po.x_shape()).astype(np.float32)
    dy = rng.standard_normal(po.y_shape()).astype(np.float32)
    dw0 = rng.standard_normal(po.w_shape()).astype(np.float32)
    want, _, _ = o.conv_backward(po, x, np.zeros(po.w_shape(), np.float32), dy, dw=dw0, want_dx=False, acc64=True)
    got = r.call(x, dy, dw0, x_off=int(operand == "x"), dy_off=int(operand == "dy"))
    assert not np.isnan(got).any()
    assert rel_err(got, want) < TOL, rel_err(got, want)


# ---- b2c_sgemm NoTrans x Trans: C (+)= A[M][K] * B[N][K]^T on the staged 1x1 kernel (one "image" of K pixels) ---------------
@pytest.mark.parametrize("K", [64, 68, 100, 4100])
@pytest.mark.parametrize("M,N", [(1, 64), (129, 65)])
@pytest.mark.parametrize("beta", [0.0, 1.0])
def test_sgemm_nt(rng, M, N, K, beta):
    L = capi.lib()
    assert L.b2c_sgemm_tc_supported(0, 1, M, N, K) == 1
    a = rng.standard_normal((M, K)).astype(np.float32)
    b = rng.standard_normal((N, K)).astype(np.float32)
    c0 = rng.standard_normal((M, N)).astype(np.float32)
    want = a.astype(np.float64) @ b.astype(np.float64).T + (c0 if beta else 0.0)
    A, B = dev(a), dev(b)
    # beta = 0 ignores C (Caffe's semantics): a NaN-filled C must not leak into the result
    Cm = dev(c0) if beta else torch.full((M, N), float("nan"), device="cuda")
    capi.sgemm(0, 1, M, N, K, 1.0, A, B, beta, Cm)
    got = host(Cm)
    assert not np.isnan(got).any()
    assert rel_err(got, want) < TOL, rel_err(got, want)
    # b2c_sgemm_ex: the split-K plan, partials in a NaN-filled workspace
    nbytes = L.b2c_sgemm_workspace_bytes(0, 1, M, N, K)
    ws = torch.full((max(nbytes, 16),), 0xFF, dtype=torch.uint8, device="cuda")
    Cx = dev(c0) if beta else torch.full((M, N), float("nan"), device="cuda")
    capi.check(L.b2c_sgemm_ex(0, 1, M, N, K, 1.0, capi._p(A), capi._p(B), beta, capi._p(Cx), capi._p(ws), nbytes,
                              capi._stream()))
    gx = host(Cx)
    assert not np.isnan(gx).any()
    assert rel_err(gx, want) < TOL, rel_err(gx, want)

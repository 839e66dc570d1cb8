"""The lo half of the tensor-core convolutions' operand splits, element by element: forward, data gradient (and its accumulating
form), weight gradient and transposed convolution, on every tensor-core route.

The schedule suites hold float data to one blob-level number (max|err| / max|ref| < 1e-4), which cannot see a lo term lost in one
K block, one N tile, one split or one image of a tile when the elements it touches are small, and their exact-integer tests have
lo = 0.  Here every case of test_conv_schedule_gpu.py, test_wgrad_schedule_gpu.py and test_deconv_gpu.py whose plan is a
tensor-core route (its regime predicate re-asserted), plus a few cases of this suite's own, runs each op through the same
harnesses (NaN workspaces, guarded or NaN-filled outputs), aligned and 4 bytes off alignment where those suites do, under two
checks (tests/tc_precision.py):
  * exact split-term probe: operands a = h + j * 2^-13 (h in {1, 2}, j in 1..7), integer bias / dx0 / dW0.  The result must
    EQUAL hi*hi' + hi*lo' + lo*hi' summed exactly (float64 oracle on the restated splits), which every partial sum holds exactly
    (max below 2^10 on the 2^-13 grid).  In TF32 math (one term, operands rounded to nearest) j is kept to 1..3, so the rounded
    operand is h and the result must equal the integer product.
  * per-element bound: normal data scaled by powers of two per image and per channel; |got - ref| <= (c_split + n 2^-23) Sum|ab|
    + 2^-23 |ref| for each element, with the split of the route that ran (ROUTE_SPLIT) and n the accumulator additions of its
    chain.  The blob-level bar still applies.  `max err / bound` is printed per run, and per route at the end of the module.
The pre-split dY buffer of the staged 3x3 weight gradient (b2c_conv_backward_filter_split) is checked next to the call without
it wherever the plan reports presplit_dy."""
import ctypes as C
import zlib
from math import ceil

import numpy as np
import pytest

import oracle as o
import tc_precision as tp
from cases import Guarded, rel_err

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import caffe_mpi_b200 as m  # noqa: E402
from caffe_mpi_b200 import capi  # noqa: E402
import deconv_oracle as do  # noqa: E402
import test_conv_schedule_gpu as cs  # noqa: E402
import test_deconv_gpu as dc  # noqa: E402
import test_wgrad_schedule_gpu as wg  # noqa: E402

FWD, BWD_DATA, BWD_FILTER = capi.OP_FORWARD, capi.OP_BACKWARD_DATA, capi.OP_BACKWARD_FILTER

# the split each tensor-core route multiplies with in the fp32 math modes, and where it was read (TF32 math: to_tf32 everywhere)
ROUTE_SPLIT = {
    "conv": {
        "staged": (tp.BF16X3, "conv_tc_stg.cu:255 split_pack_bf16 (activations); filter_prep.cu:45-47 (filter)"),
        "staged_plane": (tp.BF16X3, "conv_tc_stg.cu:255, the same converter in plane mode"),
        "gather": (tp.TF32X3, "conv_tc.cu:216 store_chunk<SPLIT> -> split_tf32; filter_prep.cu:50"),
        "gather_scatter": (tp.TF32X3, "conv_tc.cu:216, the gather kernel with the scatter epilogue"),
    },
    "wgrad": {
        "staged_3x3": (tp.BF16X3, "conv_tc_wgrad_stg.cu:176-186, 241, 267; pre-split dY :417"),
        "staged_3x3_plane": (tp.BF16X3, "conv_tc_wgrad_stg.cu:176-186, 241, 267"),
        "staged_1x1": (tp.BF16X3, "conv_tc_wgrad_stg.cu:176-186, 267"),
        "staged_1x1_plane": (tp.BF16X3, "conv_tc_wgrad_stg.cu:176-186, 267"),
        "tma_1x1": (tp.TF32X3, "conv_tc_wgrad.cu:356-357 raw tile read as truncated TF32 hi, :436 split_tf32 lo"),
        "gather": (tp.TF32X3, "conv_tc_wgrad.cu:159, 260 store_chunk<SPLIT>"),
        "compact_staged": (tp.BF16X3, "conv_tc_wgrad.cu:682-684 -> the staged 1x1 kernel on the compacted operands"),
        "compact_tma": (tp.TF32X3, "conv_tc_wgrad.cu:682-684 -> the TMA-fed 1x1 kernel on the compacted operands"),
    },
    "deconv": {
        "phase": (tp.TF32X3, "deconv.cu:10-13: one gather-kernel launch (conv_tc.cu:216) per phase"),
        "dual": (None, "deconv.cu:8: the dual convolution's own route, split per its dual_route"),
    },
}
TF32_BAR, FP32_BAR = 1e-3, 1e-4
MARGINS = {}                                 # (family, route, math) -> largest max err / bound seen


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def kind_of(family, route, math):
    if math == capi.MATH_TF32:
        return tp.TF32
    return ROUTE_SPLIT[family][route][0]


def math_name(math):
    return {None: "fp32", capi.MATH_FP32: "fp32", capi.MATH_TF32: "tf32", capi.MATH_FP32_3XTF32: "3xtf32"}[math]


def bar(math):
    return TF32_BAR if math == capi.MATH_TF32 else FP32_BAR


def probe(rng, shape, kind):
    return tp.probe_operand(rng, shape, jmax=3 if kind == tp.TF32 else 7)


def ints(rng, shape):
    return rng.integers(-4, 5, shape).astype(np.float32)


def check_probe(got, want, what):
    msg = tp.probe_mismatch(got, want)
    assert msg is None, f"{what}, exact probe: {msg}"


def check_bound(got, ref, mag, kind, n, math, what, key):
    bnd = tp.elem_bound(kind, n, mag, ref)
    worst, msg = tp.bound_report(got, ref, bnd)
    blob = rel_err(got, ref)
    print(f"[tc-precision] {what}: split {kind}, n {n}: max err / bound {worst:.3g}; blob err {blob:.3g}")
    MARGINS[key] = max(MARGINS.get(key, 0.0), worst)
    assert msg is None, f"{what}: {msg}"
    assert blob < bar(math), (what, blob)


def roundup(k, b=64):
    return -(-k // b) * b


# ---- forward and data gradient -------------------------------------------------------------------------------------------
R = cs.R

# cases only this suite has: a ragged last N tile (8 of 136 output channels on the staged kernel's 128-wide tile; 40 channels in
# a 64-wide gather tile), the scatter data gradient in TF32 math
OWN_CONV = [
    ("prec_stg_o136_ragged_tile", lambda S: cs.conv(3, 32, 8, 16, 136, 3),
     lambda q0, q1, S: R(q0, "staged", n_tile=128, n_tiles=2) and R(q1, "gather"), None, True),
    ("prec_g_o40_ragged_tile", lambda S: cs.conv(2, 16, 8, 8, 40, 3),
     lambda q0, q1, S: R(q0, "gather", n_tile=64, n_tiles=1) and R(q1, "gather"), None, True),
    ("prec_scatter_tf32", lambda S: cs.conv(2, 32, 14, 14, 40, 1, s=2),
     lambda q0, q1, S: R(q0, "gather") and R(q1, "gather_scatter"), capi.MATH_TF32, True),
    ("prec_scatter_3xtf32", lambda S: cs.conv(2, 32, 14, 14, 40, 1, s=2),
     lambda q0, q1, S: R(q0, "gather") and R(q1, "gather_scatter"), capi.MATH_FP32_3XTF32, True),
]
# the conv suite's cases with a tensor-core route (its exact-integer set: the multi-wave case is there for the schedule alone, and
# the table cliffs for the FFMA fallback)
CONV_CASES = [c for c in cs.CASES if c[4] and "cliff" not in c[0]] + OWN_CONV


def conv_ops(r, plans):
    """(op, route) for each op of the case that runs on the tensor cores"""
    return [(op, plans[op]["route"]) for op in (FWD, BWD_DATA) if plans[op]["route"] in cs.TENSOR_CORE]


@pytest.mark.parametrize("cid,shape,regime,math,exact", CONV_CASES, ids=[c[0] for c in CONV_CASES])
def test_conv_precision(rng, sms, cid, shape, regime, math, exact):
    r, plans = cs.setup(shape(sms), regime, math, sms)
    po = r.po
    ops = conv_ops(r, plans)
    assert ops, f"{cid}: no tensor-core route; plans {plans}"
    Og = po.O // po.G
    for op, route in ops:
        K = po.Kd if op == FWD else Og * po.kh * po.kw
        name = "forward" if op == FWD else "data gradient"
        for off in (0, 1):
            rt = "gather" if off and route in cs.STAGED else route          # unaligned: the staged layers take the gather kernel
            kind = kind_of("conv", rt, math)
            what = f"{cid}: {name} on route {rt} ({math_name(math)})" + (", unaligned" if off else "")
            # exact probe
            if op == FWD:
                a, w, b = probe(rng, po.x_shape(), kind), probe(rng, po.w_shape(), kind), ints(rng, po.O)
                E, a = tp.three_term(lambda u, v: o.conv_forward(po, u, v, None, acc64=True), a, w, kind)
                want = E + b[None, :, None, None]
                got = r.call(op, a, cs.dev(w), cs.dev(b), off=off)
            else:
                a, w = probe(rng, po.y_shape(), kind), probe(rng, po.w_shape(), kind)
                E, a = tp.three_term(lambda u, v: cs.oracle_dx(po, v, u), a, w, kind)
                want = E
                got = r.call(op, a, cs.dev(w), None, off=off)
            check_probe(got, want, what)
            if op == BWD_DATA and route in cs.STAGED and not off:
                dx0 = ints(rng, po.x_shape())
                acc = r.call(op, a, cs.dev(w), off=0, init=dx0, accumulate=True)
                check_probe(acc, want + dx0, what + ", accumulate")
            # per-element bound
            n = tp.chain(kind, roundup(K), extra=2)
            w = tp.pow2_scale(rng, rng.standard_normal(po.w_shape()) * (2.0 / K) ** 0.5, (0, 1))
            if op == FWD:
                a = tp.pow2_scale(rng, rng.standard_normal(po.x_shape()), (0, 1))
                b = tp.pow2_scale(rng, rng.standard_normal(po.O) * 0.1, 0)
                ref = cs.oracle_y(po, a, w, b)
                mag = cs.oracle_y(po, np.abs(a), np.abs(w), np.abs(b))
                got = r.call(op, a, cs.dev(w), cs.dev(b), off=off)
            else:
                a = tp.pow2_scale(rng, rng.standard_normal(po.y_shape()), (0, 1))
                ref = cs.oracle_dx(po, w, a)
                mag = cs.oracle_dx(po, np.abs(w), np.abs(a))
                got = r.call(op, a, cs.dev(w), None, off=off)
            check_bound(got, ref, mag, kind, n, math, what, ("conv", rt, math_name(math)))
            if op == BWD_DATA and route in cs.STAGED and not off:
                dx0 = rng.standard_normal(po.x_shape()).astype(np.float32)
                acc = r.call(op, a, cs.dev(w), off=0, init=dx0, accumulate=True)
                check_bound(acc, dx0 + ref.astype(np.float64), np.abs(dx0) + mag, kind, n + 1, math, what + ", accumulate",
                            ("conv", rt, math_name(math)))


# ---- weight gradient -----------------------------------------------------------------------------------------------------
class WRun(wg.Run):
    def call_split(self, x, dy, dw0):
        """b2c_conv_backward_filter_split with its split buffer (dY converted to bf16 hi / lo once per call): dW0 + gradient,
        NaN-filled workspace and split buffer, dW between guard bands"""
        need, sb = self.d.workspace_bytes(BWD_FILTER), self.d.wgrad_split_bytes()
        ws = torch.full((max(need, 16),), 0xFF, dtype=torch.uint8, device="cuda")
        split = torch.full((max(sb, 16),), 0xFF, dtype=torch.uint8, device="cuda")
        X, DY = cs.dev(x), cs.dev(dy)
        out = Guarded(self.n, 0, dw0)
        capi.check(capi.lib().b2c_conv_backward_filter_split(
            self.d._h, C.c_void_p(X.data_ptr()), C.c_void_p(DY.data_ptr()), out.ptr(), C.c_void_p(ws.data_ptr()), need,
            C.c_void_p(split.data_ptr()), sb, capi._stream()))
        return out.read().reshape(self.po.w_shape())


def wgrad_block_px(route):
    return 64 if route in wg.STAGED + ("compact_staged",) else 32


def wgrad_chain(kind, q, route):
    """per split: `per` K blocks of 64 (staged) or 32 (gather, TMA-fed) pixels, an accumulator fold every 8 blocks, the split
    reduction, dW0"""
    return tp.chain(kind, q["per"] * wgrad_block_px(route), q["splits"], extra=1 + ceil(q["per"] / 8))


OWN_WGRAD = [
    # the pre-split dY path of the staged 3x3 kernel, split-K boundaries inside images (3 K blocks per 12x16 image)
    ("prec_s3_presplit_mid_image", lambda S: wg.conv(20 * S // 132, 64, 12, 16, 32, 3),
     lambda q, S: q["route"] == "staged_3x3" and q["presplit_dy"] and q["splits"] > 1 and wg.mid_image_splits(q), None, True),
    # the same layer below the pre-split threshold (4 channel tiles)
    ("prec_s3_no_presplit_mid_image", lambda S: wg.conv(20 * S // 132, 32, 12, 16, 32, 3),
     lambda q, S: q["route"] == "staged_3x3" and not q["presplit_dy"] and q["splits"] > 1 and wg.mid_image_splits(q), None, True),
    # 3xTF32 math on a strided 1x1 layer: compaction, then the staged bf16x3 kernel (the split the route multiplies with)
    ("prec_compact_3xtf32", lambda S: wg.conv(20, 64, 14, 14, 40, 1, s=2),
     lambda q, S: q["route"] == "compact_staged", capi.MATH_FP32_3XTF32, True),
]
WGRAD_CASES = [c for c in wg.CASES] + OWN_WGRAD
# 4 bytes off alignment (x or dy), as the wgrad suite does: (id, case, aligned route)
WGRAD_UNALIGNED = [("staged_3x3", wg.conv(6, 16, 12, 12, 40, 3), "staged_3x3"),
                   ("tma_1x1", wg.conv(20, 48, 6, 6, 64, 1), "tma_1x1"),
                   ("compact", wg.conv(8, 32, 16, 16, 40, 1, s=2), "compact_staged")]


def wgrad_oracle(po):
    z = np.zeros(po.w_shape(), np.float32)
    return lambda u, v: o.conv_backward(po, u, z, v, want_dx=False, acc64=True)[0]


def wgrad_checks(r, rng, route, kind, n, math, what, key, x_off=0, dy_off=0, presplit=False):
    po = r.po
    f = wgrad_oracle(po)
    x, dy, dw0 = probe(rng, po.x_shape(), kind), probe(rng, po.y_shape(), kind), ints(rng, po.w_shape())
    E, x = tp.three_term(f, x, dy, kind)
    check_probe(r.call(x, dy, dw0, x_off=x_off, dy_off=dy_off), E + dw0, what)
    if presplit:
        check_probe(r.call_split(x, dy, dw0), E + dw0, what + ", pre-split dY")
    x = tp.pow2_scale(rng, rng.standard_normal(po.x_shape()), (0, 1))
    dy = tp.pow2_scale(rng, rng.standard_normal(po.y_shape()), (0, 1))
    dw0 = rng.standard_normal(po.w_shape()).astype(np.float32)
    ref = dw0 + f(x, dy).astype(np.float64)
    mag = np.abs(dw0) + f(np.abs(x), np.abs(dy)).astype(np.float64)
    check_bound(r.call(x, dy, dw0, x_off=x_off, dy_off=dy_off), ref, mag, kind, n, math, what, key)
    if presplit:
        check_bound(r.call_split(x, dy, dw0), ref, mag, kind, n, math, what + ", pre-split dY", key)


@pytest.mark.parametrize("cid,shape,regime,math,impulse", WGRAD_CASES, ids=[c[0] for c in WGRAD_CASES])
def test_wgrad_precision(rng, sms, cid, shape, regime, math, impulse):
    r = WRun(shape(sms), math)
    q = r.plan()
    assert regime(q, sms), f"{cid}: the planner no longer produces this case's regime; plan {q}"
    route = q["route"]
    kind = kind_of("wgrad", route, math)
    wgrad_checks(r, rng, route, kind, wgrad_chain(kind, q, route), math,
                 f"{cid}: weight gradient on route {route} ({math_name(math)}), plan {q}", ("wgrad", route, math_name(math)),
                 presplit=q["presplit_dy"])


@pytest.mark.parametrize("operand", ["x", "dy"])
@pytest.mark.parametrize("cid,c,route", WGRAD_UNALIGNED, ids=[u[0] for u in WGRAD_UNALIGNED])
def test_wgrad_precision_unaligned(rng, sms, cid, c, route, operand):
    """x or dy 4 bytes off alignment: compaction needs only dy aligned, everything else falls back to the gather kernel"""
    r = WRun(c)
    assert r.plan()["route"] == route
    rt = route if operand == "x" and route.startswith("compact") else "gather"
    kind = kind_of("wgrad", rt, None)
    po = r.po
    # the fallback's split plan is not reported: count every K step of the whole reduction and one split per SM
    n = tp.chain(kind, po.N * po.Ho * po.Wo, sms, extra=2 + po.N)
    wgrad_checks(r, rng, rt, kind, n, None, f"{cid}: weight gradient, {operand} unaligned, route {rt}", ("wgrad", rt, "fp32"),
                 x_off=int(operand == "x"), dy_off=int(operand == "dy"))


# ---- transposed convolution ------------------------------------------------------------------------------------------------
def deconv_setup(case, math):
    _, N, Cc, H, W, O, k, s, p, d, G, fwd_route = case
    desc = capi.DeconvDesc(dc._params(N, Cc, H, W, O, k, s, p, d, G, True), math=math)
    plans = [desc.plan(op) for op in (FWD, BWD_DATA, BWD_FILTER)]
    assert plans[0]["route"] == fwd_route, plans[0]
    assert plans[1]["route"] == "dual" and plans[2]["route"] == "dual", plans
    Ht, Wt = desc.out_shape()
    dual = m.ConvDesc(dc._params(N, O, Ht, Wt, Cc, k, s, p, d, G, False), math=math)
    qw = dual.wgrad_plan()
    assert capi.WGRAD_ROUTES[plans[2]["dual_route"]] == qw["route"], (plans[2], qw)
    routes = [("deconv", "phase") if fwd_route == "phase" else ("conv", capi.CONV_ROUTES[plans[0]["dual_route"]]),
              ("conv", capi.CONV_ROUTES[plans[1]["dual_route"]]),
              ("wgrad", qw["route"])]
    return desc, dual, qw, routes


@pytest.mark.parametrize("case", dc.TC_CASES, ids=[c[0] for c in dc.TC_CASES])
@pytest.mark.parametrize("math", [capi.MATH_FP32, capi.MATH_TF32], ids=["fp32", "tf32"])
def test_deconv_precision(case, math):
    cid, N, Cc, H, W, O, k, s, p, d, G, fwd_route = case
    rng = np.random.default_rng(zlib.crc32(("precision/" + cid).encode()))
    desc, _dual, qw, routes = deconv_setup(case, math)
    for fam, rt in routes:
        assert rt in ROUTE_SPLIT[fam] and (fam != "deconv" or rt == "phase"), (fam, rt)
    xs, ws_, ys = desc.x_shape(), desc.w_shape(), desc.y_shape()
    (kh, kw) = do._pair(k)
    taps = kh * kw
    kinds = [kind_of(fam, rt, math) for fam, rt in routes]
    mname = math_name(math)

    def fwd(x, w, b, off=0):
        Y = dc._nan(ys, off)
        desc.forward(dc._dev(x, off), dc._dev(w), None if b is None else dc._dev(b), Y)
        torch.cuda.synchronize()
        return Y.cpu().numpy()

    def bwd_data(dy, w):
        DX = dc._nan(xs)
        desc.backward_data(dc._dev(dy), dc._dev(w), DX)
        torch.cuda.synchronize()
        return DX.cpu().numpy()

    def bwd_filter(x, dy, dw0, split=False):
        DW = dc._dev(dw0)
        (desc.backward_filter_split if split else desc.backward_filter)(dc._dev(x), dc._dev(dy), DW)
        torch.cuda.synchronize()
        return DW.cpu().numpy()

    f_fwd = lambda u, v: do.deconv_forward(u, v, None, k, s, p, d, G)            # noqa: E731
    f_bd = lambda u, v: do.deconv_backward(np.zeros(xs), v, u, k, s, p, d, G)[0]   # noqa: E731
    f_bf = lambda u, v: do.deconv_backward(u, np.zeros(ws_), v, k, s, p, d, G)[1]  # noqa: E731
    presplit = qw["presplit_dy"]
    # forward, aligned and unaligned (the dual routes fall back to the gather kernel)
    for off in (0, 1):
        fam, rt = routes[0]
        if off and fam == "conv" and rt in cs.STAGED:
            rt = "gather"
        kind = kind_of(fam, rt, math)
        what = f"{cid}: deconvolution forward on {fam} route {rt} ({mname})" + (", unaligned" if off else "")
        x, w, b = probe(rng, xs, kind), probe(rng, ws_, kind), ints(rng, O)
        E, x = tp.three_term(f_fwd, x, w, kind)
        check_probe(fwd(x, w, b, off), E + b[None, :, None, None], what)
        x = tp.pow2_scale(rng, rng.standard_normal(xs), (0, 1))
        w = tp.pow2_scale(rng, rng.standard_normal(ws_) * 0.2, (0, 1))
        b = tp.pow2_scale(rng, rng.standard_normal(O), 0)
        ref = do.deconv_forward(x, w, b, k, s, p, d, G)
        mag = do.deconv_forward(np.abs(x), np.abs(w), np.abs(b), k, s, p, d, G)
        check_bound(fwd(x, w, b, off), ref, mag, kind, tp.chain(kind, roundup(Cc // G * taps), extra=2), math, what,
                    (fam, rt, mname))
    # data gradient: the dual's forward
    fam, rt = routes[1]
    kind = kinds[1]
    what = f"{cid}: deconvolution data gradient on {fam} route {rt} ({mname})"
    dy, w = probe(rng, ys, kind), probe(rng, ws_, kind)
    E, dy = tp.three_term(f_bd, dy, w, kind)
    check_probe(bwd_data(dy, w), E, what)
    dy = tp.pow2_scale(rng, rng.standard_normal(ys), (0, 1))
    w = tp.pow2_scale(rng, rng.standard_normal(ws_) * 0.2, (0, 1))
    check_bound(bwd_data(dy, w), f_bd(dy, w), f_bd(np.abs(dy), np.abs(w)), kind,
                tp.chain(kind, roundup(O // G * taps), extra=2), math, what, (fam, rt, mname))
    # weight gradient into dW0: the dual's, with X = top diff and dY = bottom data
    fam, rt = routes[2]
    kind = kinds[2]
    what = f"{cid}: deconvolution weight gradient on {fam} route {rt} ({mname}), dual plan {qw}"
    x, dy, dw0 = probe(rng, xs, kind), probe(rng, ys, kind), ints(rng, ws_)
    E, x = tp.three_term(f_bf, x, dy, kind)
    check_probe(bwd_filter(x, dy, dw0), E + dw0, what)
    if presplit:
        check_probe(bwd_filter(x, dy, dw0, split=True), E + dw0, what + ", pre-split")
    x = tp.pow2_scale(rng, rng.standard_normal(xs), (0, 1))
    dy = tp.pow2_scale(rng, rng.standard_normal(ys), (0, 1))
    dw0 = rng.standard_normal(ws_).astype(np.float32)
    ref = dw0 + f_bf(x, dy)
    mag = np.abs(dw0) + f_bf(np.abs(x), np.abs(dy))
    n = wgrad_chain(kind, qw, rt)
    check_bound(bwd_filter(x, dy, dw0), ref, mag, kind, n, math, what, (fam, rt, mname))
    if presplit:
        check_bound(bwd_filter(x, dy, dw0, split=True), ref, mag, kind, n, math, what + ", pre-split", (fam, rt, mname))


# ---- every tensor-core route is reached ------------------------------------------------------------------------------------
def routes_reached(sms):
    """{math name: {family: set of routes}} over every case of this module, from the plan queries alone"""
    seen = {}

    def add(math, fam, rt):
        seen.setdefault(math_name(math), {}).setdefault(fam, set()).add(rt)

    for cid, shape, regime, math, _ in CONV_CASES:
        r = cs.Run(shape(sms), math)
        for op, rt in conv_ops(r, r.plans()):
            add(math, "conv", rt)
    for cid, shape, regime, math, _ in WGRAD_CASES:
        q = WRun(shape(sms), math).plan()
        add(math, "wgrad", q["route"])
        if q["presplit_dy"]:
            add(math, "wgrad", q["route"] + "+presplit_dy")
    for case in dc.TC_CASES:
        for math in (capi.MATH_FP32, capi.MATH_TF32):
            _, _, _, routes = deconv_setup(case, math)
            add(math, "deconv", case[-1])
            for fam, rt in routes:
                add(math, fam, rt)
    return seen


def test_every_tensor_core_route_is_reached(sms):
    seen = routes_reached(sms)
    for mname in sorted(seen):
        for fam in sorted(seen[mname]):
            print(f"[tc-precision] {mname} {fam}: {sorted(seen[mname][fam])}")
    fp32 = seen["fp32"]
    for fam in ("conv", "wgrad"):
        missing = set(ROUTE_SPLIT[fam]) - fp32[fam]
        assert not missing, f"fp32 math: no case reaches the {fam} routes {sorted(missing)}"
    assert {"phase", "dual"} <= fp32["deconv"]
    assert {"staged_3x3+presplit_dy", "staged_3x3"} <= fp32["wgrad"]
    # TF32 math: the planners take the gather kernels (conv_route, tc_wgrad_route) and the phase / dual deconvolution routes
    tf32 = seen["tf32"]
    assert {"gather", "gather_scatter"} <= tf32["conv"] and "gather" in tf32["wgrad"] and {"phase", "dual"} <= tf32["deconv"]
    # 3xTF32 math: the gather kernels, and the compaction route of strided 1x1 weight gradients
    x3 = seen["3xtf32"]
    assert {"gather", "gather_scatter"} <= x3["conv"] and "compact_staged" in x3["wgrad"]


def test_margins_per_route():
    """the largest max err / bound per route over the runs above (printed with -s): every ratio is below 1"""
    if not MARGINS:
        pytest.skip("no precision case ran in this session")
    for (fam, rt, mname), v in sorted(MARGINS.items()):
        print(f"[tc-precision] max err / bound  {fam:6s} {rt:18s} {mname:6s} {v:.3g}")
    assert max(MARGINS.values()) <= 1.0

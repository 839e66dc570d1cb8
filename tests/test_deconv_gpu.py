"""Transposed convolution and Crop on the H100, per element against tests/deconv_oracle.py.

Each case first pins its route through b2c_debug_deconv_plan, then runs the entry point into a NaN-filled buffer (so an output
the kernels never write shows up) and compares:
  * tensor-core routes (phase route, the dual's gather / staged routes): max|err| / max|ref| against the float64 oracle at the
    convolution suites' blob-level bar, 1e-4 in the fp32 math mode and 1e-3 in TF32;
  * depthwise forward and data gradient: bit-exact against the float32 restatements of the kernels' tap order;
  * depthwise weight gradient: the same bits on repeated calls, and within the fp32 bar of float64;
  * engine CAFFE forward: bit-identical to b2c_conv_backward_data of the dual convolution (no bias);
  * Crop: bit-exact, 16-byte and scalar paths.
"""
import zlib

import numpy as np
import pytest

torch = pytest.importorskip("torch")

import caffe_mpi_b200 as m  # noqa: E402
from caffe_mpi_b200 import capi  # noqa: E402
import deconv_oracle as do  # noqa: E402

pytestmark = pytest.mark.gpu

FP32_BAR, TF32_BAR = 1e-4, 1e-3


def _err(got, ref):
    got = got.detach().cpu().numpy().astype(np.float64)
    assert not np.isnan(got).any(), "an output element was never written"
    return float(np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-30))


def _dev(a, offset=0):
    """a CUDA copy of `a`; offset > 0 places it `offset` floats into a larger buffer (4-byte but not 16-byte aligned)."""
    flat = torch.full((a.size + offset,), float("nan"), device="cuda")
    t = flat[offset:].view(a.shape)
    t.copy_(torch.from_numpy(np.ascontiguousarray(a, np.float32)))
    return t


def _nan(shape, offset=0):
    return torch.full((int(np.prod(shape)) + offset,), float("nan"), device="cuda")[offset:].view(shape)


def _params(N, Cc, H, W, O, k, s, p, d, G, bias):
    kh, kw = do._pair(k); sh, sw = do._pair(s); ph, pw = do._pair(p); dh, dw = do._pair(d)
    q = m.ConvParams.make(N, Cc, H, W, O, kh, sh, ph, dh, G, bias)
    q.kw, q.sw, q.pw, q.dw = kw, sw, pw, dw
    return q


# (name, N, C, H, W, O, k, s, p, d, G, forward route)
TC_CASES = [
    ("dcgan_4x4s2p1", 8, 64, 8, 8, 32, 4, 2, 1, 1, 1, "phase"),
    ("3x3s2p1", 4, 32, 7, 7, 16, 3, 2, 1, 1, 1, "phase"),
    ("3x3s2p0_odd", 3, 12, 5, 6, 20, 3, 2, 0, 1, 1, "phase"),
    ("k2_below_s3", 2, 16, 5, 5, 8, 2, 3, 0, 1, 1, "phase"),
    ("dilated_3x3s2d2", 2, 16, 6, 6, 24, 3, 2, 2, 2, 1, "phase"),
    ("grouped_4x4s2", 2, 16, 6, 6, 8, 4, 2, 1, 1, 2, "phase"),
    ("rect_3x5_s2x3", 2, 8, 5, 4, 12, (3, 5), (2, 3), (1, 2), 1, 1, "phase"),
    ("stride1_3x3", 2, 32, 9, 9, 16, 3, 1, 1, 1, 1, "dual"),
    ("1x1s2", 2, 32, 6, 6, 16, 1, 2, 0, 1, 1, "dual"),
    ("stride_2x1", 2, 16, 5, 6, 12, 3, (2, 1), 1, 1, 1, "phase"),        # out_ws == 1 on the phase route
    ("k5s5_25_phases", 2, 8, 4, 4, 8, 5, 5, 1, 1, 1, "phase"),           # more phases than one filter-prep launch takes (24)
]


@pytest.mark.parametrize("case", TC_CASES, ids=[c[0] for c in TC_CASES])
@pytest.mark.parametrize("math", [capi.MATH_FP32, capi.MATH_TF32], ids=["fp32", "tf32"])
def test_tensor_core_routes_against_float64(case, math):
    _, N, Cc, H, W, O, k, s, p, d, G, fwd_route = case
    rng = np.random.default_rng(zlib.crc32(case[0].encode()))
    desc = capi.DeconvDesc(_params(N, Cc, H, W, O, k, s, p, d, G, True), math=math)
    plan = desc.plan(capi.OP_FORWARD)
    assert plan["route"] == fwd_route, plan
    if fwd_route == "dual":
        assert capi.CONV_ROUTES[plan["dual_route"]] in ("staged", "gather", "gather_scatter")
    else:
        assert plan["phases"] == desc.params.sh * desc.params.sw
    bar = FP32_BAR if math == capi.MATH_FP32 else TF32_BAR
    x = rng.standard_normal(desc.x_shape()).astype(np.float32)
    w = (rng.standard_normal(desc.w_shape()) * 0.2).astype(np.float32)
    b = rng.standard_normal(O).astype(np.float32)
    y_ref = do.deconv_forward(x, w, b, k, s, p, d, G)
    dy = rng.standard_normal(y_ref.shape).astype(np.float32)
    dx_ref, dw_ref, db_ref = do.deconv_backward(x, w, dy, k, s, p, d, G)
    X, Wt, B, DY = _dev(x), _dev(w), _dev(b), _dev(dy)
    Y = _nan(y_ref.shape)
    desc.forward(X, Wt, B, Y)
    DX = _nan(x.shape)
    desc.backward_data(DY, Wt, DX)
    dw0 = rng.standard_normal(w.shape).astype(np.float32)
    DW, DB = _dev(dw0), _dev(np.zeros(O, np.float32))
    desc.backward_filter(X, DY, DW)
    desc.backward_bias(DY, DB)
    torch.cuda.synchronize()
    assert _err(Y, y_ref) < bar
    assert _err(DX, dx_ref) < bar
    assert _err(DW, dw_ref + dw0) < bar
    assert _err(DB, db_ref) < 1e-5
    # unaligned activations (4-byte aligned only): the phase route runs the same gather launches, so the same bits; the dual
    # routes fall back as the convolution routes do
    Xu, Yu = _dev(x, 1), _nan(y_ref.shape, 1)
    desc.forward(Xu, Wt, B, Yu)
    torch.cuda.synchronize()
    if fwd_route == "phase":
        assert torch.equal(Yu, Y)
    assert _err(Yu, y_ref) < bar


def test_split_weight_gradient_matches_plain():
    desc = capi.DeconvDesc(_params(4, 64, 8, 8, 64, 3, 1, 1, 1, 1, False))
    rng = np.random.default_rng(5)
    x = rng.standard_normal(desc.x_shape()).astype(np.float32)
    dy = rng.standard_normal(desc.y_shape()).astype(np.float32)
    X, DY = _dev(x), _dev(dy)
    A, Bv = _dev(np.zeros(desc.w_shape(), np.float32)), _dev(np.zeros(desc.w_shape(), np.float32))
    desc.backward_filter(X, DY, A)
    desc.backward_filter_split(X, DY, Bv)
    torch.cuda.synchronize()
    assert torch.equal(A, Bv)
    _, dw_ref, _ = do.deconv_backward(x, np.zeros(desc.w_shape()), dy, 3, 1, 1, 1)
    assert _err(A, dw_ref) < FP32_BAR


def test_caffe_engine_is_the_dual_data_gradient():
    # engine CAFFE: per-image GEMM + col2im of the dual, bit for bit; the bias pass adds once
    N, Cc, H, O, k, s, p = 3, 6, 5, 4, 3, 2, 1
    desc = capi.DeconvDesc(_params(N, Cc, H, H, O, k, s, p, 1, 1, True), capi.ENGINE_CAFFE)
    assert desc.plan(0)["route"] == "dual" and capi.CONV_ROUTES[desc.plan(0)["dual_route"]] == "caffe"
    Ht, Wt = desc.out_shape()
    dual = m.ConvDesc(m.ConvParams.make(N, O, Ht, Wt, Cc, k, s, p, 1, 1, False), capi.ENGINE_CAFFE)
    rng = np.random.default_rng(6)
    x = rng.standard_normal(desc.x_shape()).astype(np.float32)
    w = rng.standard_normal(desc.w_shape()).astype(np.float32)
    b = rng.standard_normal(O).astype(np.float32)
    X, Wd, B = _dev(x), _dev(w), _dev(b)
    Y, Yd = _nan(desc.y_shape()), _nan(desc.y_shape())
    nob = capi.DeconvDesc(_params(N, Cc, H, H, O, k, s, p, 1, 1, False), capi.ENGINE_CAFFE)
    nob.forward(X, Wd, None, Y)
    dual.backward_data(X, Wd, Yd)
    torch.cuda.synchronize()
    assert torch.equal(Y, Yd)
    desc.forward(X, Wd, B, Y)
    torch.cuda.synchronize()
    assert torch.equal(Y, Yd + B.view(1, -1, 1, 1))
    assert _err(Y, do.deconv_forward(x, w, b, k, s, p, 1)) < 1e-5


# ---- depthwise (group == C == num_output) ----------------------------------------------------------------------------------
DW_CASES = [  # (name, N, C, H, k, s, p, d)
    ("bilinear_x2", 4, 16, 9, 4, 2, 1, 1),
    ("3x3s2", 2, 8, 7, 3, 2, 0, 1),
    ("k2_below_s3", 2, 4, 5, 2, 3, 0, 1),
    ("dilated", 2, 4, 6, 3, 2, 1, 2),
    ("fcn_64s32", 1, 21, 8, 64, 32, 16, 1),
]


@pytest.mark.parametrize("case", DW_CASES, ids=[c[0] for c in DW_CASES])
@pytest.mark.parametrize("offset", [0, 1], ids=["aligned", "unaligned"])
def test_depthwise_kernels(case, offset):
    _, N, Cc, H, k, s, p, d = case
    desc = capi.DeconvDesc(_params(N, Cc, H, H, Cc, k, s, p, d, Cc, True))
    for op in (0, 1, 2):
        assert desc.plan(op)["route"] == "depthwise"
    rng = np.random.default_rng(7)
    x = rng.standard_normal(desc.x_shape()).astype(np.float32)
    w = do.bilinear_weights(desc.w_shape()) if case[0].startswith(("bilinear", "fcn")) else \
        rng.standard_normal(desc.w_shape()).astype(np.float32)
    w = w + rng.standard_normal(w.shape).astype(np.float32) * np.float32(0.01)
    b = rng.standard_normal(Cc).astype(np.float32)
    X, Wd, B = _dev(x, offset), _dev(w, offset), _dev(b, offset)
    Y = _nan(desc.y_shape(), offset)
    desc.forward(X, Wd, B, Y)
    dy = rng.standard_normal(desc.y_shape()).astype(np.float32)
    DY = _dev(dy, offset)
    DX = _nan(x.shape, offset)
    desc.backward_data(DY, Wd, DX)
    dw0 = rng.standard_normal(w.shape).astype(np.float32)
    DW1, DW2 = _dev(dw0, offset), _dev(dw0, offset)
    desc.backward_filter(X, DY, DW1)
    desc.backward_filter(X, DY, DW2)
    torch.cuda.synchronize()
    assert np.array_equal(Y.cpu().numpy(), do.dw_forward_f32(x, w, b, k, s, p, d))
    assert np.array_equal(DX.cpu().numpy(), do.dw_dgrad_f32(dy, w, H, H, k, s, p, d))
    assert torch.equal(DW1, DW2)
    _, dw_ref, _ = do.deconv_backward(x, w, dy, k, s, p, d, G=Cc)
    assert _err(DW1, dw_ref + dw0) < FP32_BAR
    assert _err(Y, do.deconv_forward(x, w, b, k, s, p, d, G=Cc)) < 1e-5


# ---- Crop ------------------------------------------------------------------------------------------------------------------
CROP_CASES = [  # (bottom, ref, axis, offset)
    ((2, 4, 5, 4), (2, 3, 4, 2), 0, ()),
    ((2, 4, 5, 4), (2, 3, 4, 2), 0, (0, 1, 1, 2)),
    ((2, 4, 5, 4), (2, 3, 4, 2), 2, (1, 2)),
    ((2, 4, 5, 4, 2), (2, 3, 4, 2, 1), 2, (1, 2, 0)),
    ((3, 8, 37, 40), (3, 8, 32, 32), 2, (3, 4)),      # 16-byte units
    ((3, 8, 37, 40), (3, 8, 32, 32), 2, (3, 5)),      # innermost offset breaks them
]


@pytest.mark.parametrize("case", CROP_CASES)
@pytest.mark.parametrize("offset", [0, 1], ids=["aligned", "unaligned"])
def test_crop_bit_exact(case, offset):
    bshape, rshape, axis, off = case
    top, offs = do.crop_offsets(bshape, rshape, axis, off)
    rng = np.random.default_rng(8)
    x = rng.standard_normal(bshape).astype(np.float32)
    g = rng.standard_normal(top).astype(np.float32)
    X, T = _dev(x, offset), _nan(top, offset)
    capi.crop_forward(X, T, offs)
    G, DX = _dev(g, offset), _nan(bshape, offset)
    capi.crop_backward(G, DX, offs)
    torch.cuda.synchronize()
    assert np.array_equal(T.cpu().numpy(), do.crop_forward(x, top, offs))
    assert np.array_equal(DX.cpu().numpy(), do.crop_backward(g, bshape, offs))


# ---- whole net: Convolution -> Deconvolution -> Crop, a frozen bilinear upsampler, Eltwise SUM, SigmoidCrossEntropyLoss ---------
from caffe_mpi_b200 import host_api  # noqa: E402


@pytest.mark.parametrize("variant", ["2d", "force_nd", "caffe_engine"])
def test_encoder_decoder_net_against_the_oracle(variant):
    N = 4
    net = do.encdec_prototxt(N, force_nd=variant == "force_nd", engine="CAFFE" if variant == "caffe_engine" else "")
    lr, mom = 0.1, 0.9
    t = host_api.Trainer(net, f'base_lr: {lr} lr_policy: "fixed" momentum: {mom} max_iter: 10', num_classes=2)
    rng = np.random.default_rng(21)
    shapes = [(6, 3, 3, 3), (6,), (6, 3, 4, 4), (3,), (6, 1, 4, 4), (3, 6, 1, 1), (3,)]
    bil = t.get_param(4, 0).reshape(shapes[4])
    assert np.array_equal(bil, do.bilinear_weights(shapes[4]))              # the "bilinear" filler, bit for bit
    params = [(rng.standard_normal(s) * 0.3).astype(np.float32) for s in shapes]
    params[4] = bil
    for i, p in enumerate(params):
        if i != 4:
            t.set_param(i, p)
    data = rng.standard_normal((N, 3, 8, 8)).astype(np.float32)
    target = rng.uniform(0, 1, (N, 192)).astype(np.float32)
    t.set_blob("data", data)
    t.set_blob("target", target)
    loss = t.forward_backward()
    ref_loss, grads, blobs = do.encdec_forward_backward(params, data, target)
    assert abs(loss - ref_loss) <= 1e-5 * abs(ref_loss), (loss, ref_loss)
    for nm in ("up", "crop", "bil", "sum"):
        assert _err(torch.from_numpy(t.get_blob(nm).reshape(blobs[nm].shape)), blobs[nm]) < FP32_BAR, nm
    for i, g in enumerate(grads):
        if i == 4:
            continue                                                         # lr_mult 0: never applied
        assert _err(torch.from_numpy(t.get_param(i, 1).reshape(g.shape)), g) < FP32_BAR, i
    # three SGD steps against the oracle; the frozen upsampler keeps its bits
    ws = [p.astype(np.float64) for p in params]
    hs = [np.zeros_like(w) for w in ws]
    for _ in range(3):
        _, gs, _ = do.encdec_forward_backward(ws, data, target)
        for i in range(len(ws)):
            if i == 4:
                continue
            hs[i] = mom * hs[i] + lr * gs[i]
            ws[i] = ws[i] - hs[i]
    t.clear_param_diffs()
    t.step(3)
    for i, w in enumerate(ws):
        got = t.get_param(i, 0).reshape(w.shape)
        if i == 4:
            assert np.array_equal(got, bil)
        else:
            assert _err(torch.from_numpy(got), w) < 1e-4, i

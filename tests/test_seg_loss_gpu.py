"""SoftmaxWithLoss and Accuracy over spatial positions on the device: b2c_softmax_loss_forward_ex / _backward_ex and
b2c_accuracy_ex against the float64 oracle of tests/seg_oracle.py, each case with its route pinned by
b2c_debug_softmax_loss_plan and its outputs NaN-filled before the call; then a small segmentation net through TrainNet."""
import numpy as np
import pytest
import torch

import seg_oracle as so
from caffe_mpi_b200 import capi, host_api

pytestmark = pytest.mark.gpu

IGN = 255


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def nan_like(shape, offset=0):
    """A NaN-filled float32 device tensor of `shape`, starting `offset` floats into its allocation (offset 1: misaligned)."""
    n = int(np.prod(shape))
    buf = torch.full((n + 4,), float("nan"), device="cuda")
    return buf[offset:offset + n].view(*shape)


def make_case(shape, axis, ignore, seed, oob=False):
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal(shape) * 3).astype(np.float32)
    outer, C, inner = so.view(shape, axis)
    lab = rng.integers(0, C, outer * inner).astype(np.float32)
    if ignore == "some":
        lab[rng.random(lab.size) < 0.3] = IGN
    elif ignore == "all":
        lab[:] = IGN
    if oob:
        lab[1] = C + 3                                                         # out of range and not ignored
        lab[-1] = -2
    return x, lab, (outer, C, inner)


# (shape, axis, route): C in {1, 2, 5, 21, 150}, inner in {1, 3, 4, 6, 4097, 512*512}
SHAPES = [
    ((64, 5), 1, "row"),
    ((256, 150), 1, "row"),
    ((7, 1, 3), 1, "column"),
    ((6, 2, 4), 1, "column_f4"),
    ((10, 5, 2, 3), 1, "column"),
    ((3, 21, 4097), 1, "column"),
    ((2, 21, 512, 512), 1, "column_f4"),
    ((4, 3, 5, 21), 2, "column"),                 # axis 2: outer 12, inner 21
    ((2, 6, 8, 21), -1, "row"),                   # NHWC with axis -1: inner 1
    ((2, 150, 16, 16), 1, "column_f4"),
]


@pytest.mark.parametrize("norm", ["VALID", "FULL", "BATCH_SIZE", "NONE"])
@pytest.mark.parametrize("ignore", [None, "some", "all"])
@pytest.mark.parametrize("case", range(len(SHAPES)))
def test_softmax_loss_forward_backward(case, ignore, norm):
    shape, axis, route = SHAPES[case]
    if ignore == "all" and norm != "VALID" and case % 3:
        pytest.skip("every-label-ignored is covered at VALID and on a third of the shapes")
    x, lab, (outer, C, inner) = make_case(shape, axis, ignore, seed=case * 7 + 1)
    ign = IGN if ignore else None
    X, L = dev(x), dev(lab)
    P = nan_like(x.shape)
    q = capi.softmax_loss_plan(outer, C, inner, X.data_ptr(), P.data_ptr())
    assert q["route"] == route
    ws = torch.empty(q["workspace"] // 4, device="cuda")
    loss, nrm = nan_like((1,)), nan_like((1,))
    capi.softmax_loss_forward_ex(outer, C, inner, X, L, P, loss, nrm, ws, ignore_label=ign, norm=norm)
    # prob is b2c_softmax_forward's, bit for bit
    Y = nan_like(x.shape)
    capi.check(capi.lib().b2c_softmax_forward(outer, C, inner, capi._p(X), capi._p(Y), capi._stream()))
    torch.cuda.synchronize()
    assert torch.equal(P.view(-1).view(torch.int32), Y.view(-1).view(torch.int32))
    want, want_n, _, _ = so.softmax_loss(x, lab, axis=axis, ignore_label=ign, norm=norm)
    got = float(loss.item())
    assert float(nrm.item()) == want_n
    assert abs(got - want) <= 1e-6 * abs(want), (got, want)
    # the same bits on a repeated call
    loss2 = nan_like((1,))
    capi.softmax_loss_forward_ex(outer, C, inner, X, L, P, loss2, nrm, ws, ignore_label=ign, norm=norm)
    torch.cuda.synchronize()
    assert loss2.view(torch.int32).item() == loss.view(torch.int32).item()
    for lw in (0.5, 3.0):
        DX = nan_like(x.shape)
        capi.softmax_loss_backward_ex(outer, C, inner, P, L, nrm, lw, DX, ignore_label=ign)
        torch.cuda.synchronize()
        p = P.cpu().numpy().reshape(outer, C, inner)
        li = lab.reshape(outer, inner).astype(np.int64)
        s = np.float32(np.float32(lw) / np.float32(want_n))
        onehot = (np.arange(C)[None, :, None] == li[:, None, :]).astype(np.float32)
        ref = ((p - onehot) * s).astype(np.float32)
        if ign is not None:
            ref = np.where((li == ign)[:, None, :], np.float32(0), ref)
        assert np.array_equal(DX.cpu().numpy().reshape(outer, C, inner), ref)


@pytest.mark.parametrize("inner,offset", [(4, 0), (4, 1), (8, 1), (6, 0)])
def test_misaligned_pointers_take_the_scalar_column(inner, offset):
    x, lab, (outer, C, _) = make_case((3, 5, inner), 1, "some", seed=inner + offset)
    X = nan_like(x.shape, offset)
    X.copy_(dev(x))
    P, L = nan_like(x.shape, offset), dev(lab)
    q = capi.softmax_loss_plan(outer, C, inner, X.data_ptr(), P.data_ptr())
    assert q["route"] == ("column_f4" if inner % 4 == 0 and offset == 0 else "column")
    ws = torch.empty(q["workspace"] // 4, device="cuda")
    loss, nrm = nan_like((1,)), nan_like((1,))
    capi.softmax_loss_forward_ex(outer, C, inner, X, L, P, loss, nrm, ws, ignore_label=IGN)
    DX = nan_like(x.shape, offset)
    capi.softmax_loss_backward_ex(outer, C, inner, P, L, nrm, 1.0, DX, ignore_label=IGN)
    torch.cuda.synchronize()
    want, _, _, dx = so.softmax_loss(x, lab, ignore_label=IGN)
    assert abs(loss.item() - want) <= 1e-6 * abs(want)
    assert np.allclose(DX.cpu().numpy(), dx, rtol=1e-5, atol=1e-7)


def test_out_of_range_label_stays_in_bounds():
    """A label outside [0, C) that is not ignored: the loss reads the nearest class, the backward subtracts nothing, accuracy
    counts a miss and touches no per-class counter.  Neighbouring memory is left alone."""
    for shape in ((12, 5), (3, 5, 8)):
        x, lab, (outer, C, inner) = make_case(shape, 1, None, seed=5, oob=True)
        X, L = dev(x), dev(lab)
        guard = torch.full((x.size + 64,), 7.0, device="cuda")
        P = guard[32:32 + x.size].view(*shape)
        q = capi.softmax_loss_plan(outer, C, inner, X.data_ptr(), P.data_ptr())
        ws = torch.empty(q["workspace"] // 4, device="cuda")
        loss, nrm = nan_like((1,)), nan_like((1,))
        capi.softmax_loss_forward_ex(outer, C, inner, X, L, P, loss, nrm, ws, ignore_label=IGN)
        dguard = torch.full((x.size + 64,), 7.0, device="cuda")
        DX = dguard[32:32 + x.size].view(*shape)
        capi.softmax_loss_backward_ex(outer, C, inner, P, L, nrm, 1.0, DX, ignore_label=IGN)
        acc, pc = nan_like((1,)), nan_like((C,))
        scratch = torch.empty(2 + 2 * C, dtype=torch.int32, device="cuda")
        capi.accuracy_ex(outer, C, inner, 1, X, L, acc, pc, scratch, ignore_label=IGN)
        torch.cuda.synchronize()
        want, _, _, dx = so.softmax_loss(x, lab, ignore_label=IGN)
        assert abs(loss.item() - want) <= 1e-6 * abs(want)
        assert np.allclose(DX.cpu().numpy(), dx, rtol=1e-5, atol=1e-7)
        for g in (guard, dguard):
            assert torch.all(g[:32] == 7.0) and torch.all(g[32 + x.size:] == 7.0)
        wa, wpc = so.accuracy(x, lab, top_k=1, ignore_label=IGN)
        assert acc.item() == wa and np.array_equal(pc.cpu().numpy(), wpc)


ACC_SHAPES = [((100, 10), 1), ((2, 10, 4, 5), 1), ((7, 2, 3), 1), ((4, 21, 4097), 1), ((3, 6, 5, 150), -1), ((2, 150, 9, 9), 1),
              ((2, 1, 6), 1), ((5, 4, 3, 2), 2)]


@pytest.mark.parametrize("ignore", [None, "some", "all"])
@pytest.mark.parametrize("top_k", [1, 3])
@pytest.mark.parametrize("case", range(len(ACC_SHAPES)))
def test_accuracy_ex(case, top_k, ignore):
    shape, axis = ACC_SHAPES[case]
    x, lab, (outer, C, inner) = make_case(shape, axis, ignore, seed=case + 40)
    top_k = min(top_k, C)
    x = np.round(x).astype(np.float32)                                         # many ties: the larger index ranks first
    ign = IGN if ignore else None
    X, L = dev(x), dev(lab)
    acc, pc = nan_like((1,)), nan_like((C,))
    scratch = torch.empty(2 + 2 * C, dtype=torch.int32, device="cuda")
    capi.accuracy_ex(outer, C, inner, top_k, X, L, acc, pc, scratch, ignore_label=ign)
    acc2 = nan_like((1,))
    capi.accuracy_ex(outer, C, inner, top_k, X, L, acc2, None, scratch, ignore_label=ign)
    torch.cuda.synchronize()
    wa, wpc = so.accuracy(x, lab, axis=axis, top_k=top_k, ignore_label=ign)
    if ignore == "all":
        assert np.isnan(acc.item()) and np.isnan(acc2.item())
    else:
        assert acc.item() == wa and acc2.item() == wa
    assert np.array_equal(pc.cpu().numpy(), wpc)


# ---- through TrainNet ---------------------------------------------------------------------------------------------------------
def rel(a, b):
    return float(np.abs(np.asarray(a, np.float64) - b).max() / max(np.abs(b).max(), 1e-30))


@pytest.mark.parametrize("norm", ["", "normalize: false", "normalization: FULL"])
def test_fcn_through_trainnet(norm):
    """conv -> pool -> conv -> Deconvolution (bilinear, lr_mult 0) -> Crop -> SoftmaxWithLoss (ignore_label, prob top) and Accuracy
    (per-class top) through TrainNet against the float64 net oracle: loss, blobs, prob, both accuracy tops exactly on the net's own
    scores, every parameter gradient and three SGD steps with momentum."""
    import deconv_oracle as do
    N, H, W, C = 4, 8, 10, 5
    mode = {"": "VALID", "normalize: false": "BATCH_SIZE", "normalization: FULL": "FULL"}[norm]
    lr, mom = 0.1, 0.9
    solver = f'base_lr: {lr} lr_policy: "fixed" momentum: {mom} max_iter: 10'
    t = host_api.Trainer(so.fcn_prototxt(N, H, W, C, norm), solver, num_classes=C)
    rng = np.random.default_rng(3)
    shapes = so.fcn_param_shapes(C)
    bil = t.get_param(4, 0).reshape(shapes[4])
    assert np.array_equal(bil, do.bilinear_weights(shapes[4]))
    params = [(rng.standard_normal(sh) * 0.5).astype(np.float32) for sh in shapes]
    params[4] = bil
    for i in range(4):
        t.set_param(i, params[i])
    x = rng.standard_normal((N, 3, H, W)).astype(np.float32)
    lab = rng.integers(0, C, (N, 1, H, W)).astype(np.float32)
    lab[rng.random(lab.shape) < 0.25] = 255
    t.set_blob("data", x)
    t.set_blob("label", lab)
    loss = t.forward_backward()
    want, grads, blobs = so.fcn_forward_backward(params, x, lab, norm=mode)
    assert abs(loss - want) <= 1e-5 * abs(want), (loss, want)
    for nm in ("c1", "p1", "sc", "up", "crop", "prob"):
        assert rel(t.get_blob(nm).reshape(blobs[nm].shape), blobs[nm]) < 1e-5, nm
    crop = t.get_blob("crop").reshape(blobs["crop"].shape)
    wa, wpc = so.accuracy(crop, lab, ignore_label=255)                # exact, on the scores the net computed
    assert t.get_blob("acc")[0] == wa
    assert np.array_equal(t.get_blob("per_class"), wpc) and wpc.max() > 0
    for i in range(4):
        assert rel(t.get_param(i, 1).reshape(grads[i].shape), grads[i]) < 1e-4, i
    ws = [p.astype(np.float64) for p in params]
    hs = [np.zeros_like(w) for w in ws]
    for _ in range(3):
        _, gs, _ = so.fcn_forward_backward(ws, x, lab, norm=mode)
        for i in range(4):
            hs[i] = mom * hs[i] + lr * gs[i]
            ws[i] = ws[i] - hs[i]
    t.clear_param_diffs()
    t.step(3)
    for i, w in enumerate(ws):
        got = t.get_param(i, 0).reshape(w.shape)
        if i == 4:
            assert np.array_equal(got, bil)
        else:
            assert rel(got, w) < 1e-4, i


def test_softmax_loss_refuses_a_label_that_needs_a_gradient():
    """softmax_loss_layer.cpp:128-130: the label bottom cannot take a gradient -- refused when the net is built."""
    net = ('name: "bad" layer { name: "data" type: "Input" top: "data" input_param { shape { dim: 4 dim: 6 } } }\n'
           'layer { name: "a" type: "InnerProduct" bottom: "data" top: "a" inner_product_param { num_output: 3 } }\n'
           'layer { name: "b" type: "InnerProduct" bottom: "data" top: "b" inner_product_param { num_output: 1 } }\n'
           'layer { name: "loss" type: "SoftmaxWithLoss" bottom: "a" bottom: "b" top: "loss" }\n')
    with pytest.raises(host_api.HostError, match="SoftmaxWithLoss Layer cannot backpropagate to label inputs."):
        host_api.Trainer(net, 'base_lr: 0.01 lr_policy: "fixed" max_iter: 1', num_classes=3)

"""The neuron kernels on the device: b2c_neuron_forward / _backward for every kind and b2c_prelu_forward / _backward on every launch
regime b2c_debug_neuron_plan reports, in NaN-prefilled guarded buffers (cases.Guarded), aligned and 4 bytes off, in and out of
place; then a small net of every neuron layer through TrainNet against the float64 net oracle of tests/neuron_oracle.py."""
import numpy as np
import pytest
import torch

import neuron_oracle as no
from cases import Guarded
from caffe_mpi_b200 import capi, host_api

pytestmark = pytest.mark.gpu

ULP = 2.0 ** -23
# per kind: the layer parameters, a draw for x, and the bound on |got - ref| for the transcendental rules, in units of 2^-23 of
# max(|ref|, floor) (forward) or max(|ref|, floor |dy|) (backward); None: bit-exact against the float32 restatement.  ELU and BNLL
# take floor 1: the reference's own expressions (alpha (exp(x) - 1.), log(1. + exp(x)), dy (y + alpha)) cancel near the values they
# approach, and the kernels keep those expressions.
CASES = {
    "ELU": ({"alpha": 0.7}, lambda r, n: r.standard_normal(n) * 3, 4),
    "POWER_1": ({"power": 1.0, "scale": 0.83, "shift": -2.4}, lambda r, n: r.standard_normal(n), None),
    "POWER_2": ({"power": 2.0, "scale": 0.34, "shift": -2.4}, lambda r, n: r.standard_normal(n), None),
    "POWER_2s0": ({"power": 2.0, "scale": 0.5, "shift": 0.0}, lambda r, n: r.standard_normal(n), None),
    "POWER_frac": ({"power": 0.37, "scale": 0.83, "shift": 2.4}, lambda r, n: np.abs(r.standard_normal(n)) + 0.1, 8),
    "POWER_s0": ({"power": -1.5, "scale": 0.8, "shift": 0.0}, lambda r, n: np.abs(r.standard_normal(n)) + 0.5, 12),
    "ABSVAL": ({}, lambda r, n: r.standard_normal(n), None),
    "BNLL": ({}, lambda r, n: r.standard_normal(n) * 20, 4),
    "EXP": ({"base": 2.0, "scale": 0.5, "shift": 1.0}, lambda r, n: r.standard_normal(n) * 3, 16),
    "EXP_e": ({}, lambda r, n: r.standard_normal(n) * 3, 8),
    "LOG": ({"base": 10.0, "scale": 0.5, "shift": 1.5}, lambda r, n: np.abs(r.standard_normal(n)) * 3, 8),
    "LOG_e": ({}, lambda r, n: np.abs(r.standard_normal(n)) * 3 + 1e-3, 8),
    "THRESHOLD": ({"threshold": 0.3}, lambda r, n: r.standard_normal(n), None),
}


def kind_of(case):
    return case.split("_")[0]


def f32(a):
    return np.asarray(a, np.float32)


@pytest.mark.parametrize("in_place", [False, True])
@pytest.mark.parametrize("off", [0, 1])
@pytest.mark.parametrize("n", [1, 7, 4099])
@pytest.mark.parametrize("case", sorted(CASES))
def test_elementwise(case, n, off, in_place):
    kind = kind_of(case)
    q, draw, bound = CASES[case]
    rng = np.random.default_rng(n * 7 + off)
    x = f32(draw(rng, n))
    dy = f32(rng.standard_normal(n))
    pf, pb = no.kernel_params(kind, q), no.kernel_params(kind, q, backward=True)
    X = Guarded(n, off, init=x)
    Y = X if in_place else Guarded(n, off)
    capi.check(capi.lib().b2c_neuron_forward(capi.NEURON_KINDS.index(kind), n, X.ptr(), Y.ptr(), *pf, None))
    y = Y.read().copy()
    Y2 = Guarded(n, off, init=x) if in_place else Guarded(n, off)
    capi.check(capi.lib().b2c_neuron_forward(capi.NEURON_KINDS.index(kind), n, (Y2 if in_place else X).ptr(), Y2.ptr(), *pf, None))
    assert np.array_equal(Y2.read().view(np.uint32), y.view(np.uint32))      # the same bits on a second call
    with np.errstate(all="ignore"):
        ref = no.forward(kind, x.astype(np.float64), q)
    floor = 1.0 if kind in ("ELU", "BNLL") else 1e-30
    if bound is None and kind == "POWER" and pf[0] == 2 and pf[0] * pf[1] != 0:
        # powf(t, 2) as the reference's caffe_gpu_powx evaluates it: within one ulp of the rounded t * t, not always equal to it
        r = no.forward_f32(kind, x, pf)
        assert np.all(np.abs(y - r) <= np.spacing(np.abs(r))), case
    elif bound is None:
        np.testing.assert_array_equal(y, no.forward_f32(kind, x, pf))
    else:
        err = np.abs(y - ref) / np.maximum(np.abs(ref), floor)
        assert err.max() <= bound * ULP, (case, err.max() / ULP)
    if kind == "THRESHOLD":
        with pytest.raises(capi.B2CError, match="Threshold"):
            capi.check(capi.lib().b2c_neuron_backward(6, n, X.ptr(), None, X.ptr(), X.ptr(), *pb, None))
        return
    # backward: x kept separately (in place the top stands where the bottom was; only the rules reading y see it)
    Xb = Guarded(n, off, init=x)
    Yb = Guarded(n, off, init=y)
    DY = Guarded(n, off, init=dy)
    DX = DY if in_place else Guarded(n, off)
    capi.check(capi.lib().b2c_neuron_backward(capi.NEURON_KINDS.index(kind), n, Xb.ptr(), Yb.ptr(), DY.ptr(), DX.ptr(), *pb, None))
    dx = DX.read().copy()
    ref = no.backward(kind, x.astype(np.float64), dy.astype(np.float64), q)
    if bound is None:
        np.testing.assert_array_equal(dx, no.backward_f32(kind, x, y, dy, pb))
    else:
        # the reference differentiates through the float32 y (ELU, Exp, Power's y / x): its rounding enters with weight ~1
        err = np.abs(dx - ref) / np.maximum(np.abs(ref), np.maximum(floor * np.abs(dy), 1e-30))
        assert err.max() <= 2 * bound * ULP, (case, err.max() / ULP)
    DY2 = Guarded(n, off, init=dy)
    DX2 = DY2 if in_place else Guarded(n, off)
    capi.check(capi.lib().b2c_neuron_backward(capi.NEURON_KINDS.index(kind), n, Xb.ptr(), Yb.ptr(), DY2.ptr(), DX2.ptr(), *pb, None))
    assert np.array_equal(DX2.read().view(np.uint32), dx.view(np.uint32))


def test_backward_reads_only_what_its_rule_needs():
    n = 1000
    rng = np.random.default_rng(2)
    x, dy = f32(np.abs(rng.standard_normal(n)) + 0.5), f32(rng.standard_normal(n))
    X, DY = torch.from_numpy(x).cuda(), torch.from_numpy(dy).cuda()
    y = torch.exp(X)
    for kind, p, xx, yy in (("EXP", (1.0, 1.0, 0.0), None, y), ("ABSVAL", (0, 0, 0), X, None), ("BNLL", (0, 0, 0), X, None),
                            ("POWER", (1.0, 0.5, 0.0), None, None), ("POWER", (2.0, 0.5, 0.0), X, None)):
        DX = torch.full_like(X, float("nan"))
        capi.neuron_backward(kind, xx, yy, DY, DX, p)
        torch.cuda.synchronize()
        assert torch.isfinite(DX).all(), kind
    with pytest.raises(capi.B2CError, match="reads x"):
        capi.neuron_backward("LOG", None, y, DY, torch.empty_like(X), (1.0, 0.0, 1.0))
    with pytest.raises(capi.B2CError, match="reads y"):
        capi.neuron_backward("ELU", X, None, DY, torch.empty_like(X), (1.0, 0.0, 0.0))


# ---- PReLU ----------------------------------------------------------------------------------------------------------------------
# (N, C, dim): one CTA per channel with a float4 or a scalar stripe, several CTAs per channel (the stem-like maps), 1 x 1 maps
PRELU_SHAPES = [(2, 3, 5), (4, 16, 1), (8, 64, 49), (2, 512, 49), (4, 64, 56 * 56), (2, 8, 112 * 112), (3, 5, 7 * 7 + 1), (1, 2, 4),
                (16, 3, 15 * 15)]


def prelu_case(shape, shared, seed):
    N, Cc, dim = shape
    rng = np.random.default_rng(seed)
    x = f32(rng.standard_normal((N, Cc, dim)))
    x[rng.random(x.shape) < 0.05] = 0.0                                         # x == 0 takes the slope side
    slope = f32(rng.uniform(0.05, 0.5, 1 if shared else Cc))
    dy = f32(rng.standard_normal(x.shape))
    return x, slope, dy


def test_prelu_shapes_cover_every_regime():
    regimes = set()
    for shape in PRELU_SHAPES:
        for shared in (False, True):
            p = capi.neuron_plan("prelu_backward", *shape, shared=shared)
            regimes.add((p["vec"], p["blocks_per_channel"] > 1))
    assert regimes == {(False, False), (True, False), (False, True), (True, True)}


@pytest.mark.parametrize("in_place", [False, True])
@pytest.mark.parametrize("off", [0, 1])
@pytest.mark.parametrize("shared", [False, True])
@pytest.mark.parametrize("case", range(len(PRELU_SHAPES)))
def test_prelu(case, shared, off, in_place):
    shape = PRELU_SHAPES[case]
    N, Cc, dim = shape
    x, slope, dy = prelu_case(shape, shared, case * 4 + off)
    n = x.size
    S = torch.from_numpy(slope).cuda()
    X = Guarded(n, off, init=x)
    Y = X if in_place else Guarded(n, off)
    K = Guarded(n, off) if in_place else None
    capi.check(capi.lib().b2c_prelu_forward(N, Cc, dim, int(shared), X.ptr(), capi._p(S), Y.ptr(), K.ptr() if K else None, None))
    np.testing.assert_array_equal(Y.read(), no.prelu_forward_f32(x.reshape(N, Cc, dim), slope, shared).reshape(-1))
    if K:
        np.testing.assert_array_equal(K.read(), x.reshape(-1))
    ws = torch.zeros(max(1, capi.prelu_workspace_bytes(N, Cc, dim, shared)), dtype=torch.uint8, device="cuda")
    Xin = K if K else X
    dx_ref, ds_ref, mag = no.prelu_backward(x.reshape(N, Cc, dim), dy.reshape(N, Cc, dim), slope, shared)
    dx_f32 = no.prelu_dx_f32(x.reshape(N, Cc, dim), dy.reshape(N, Cc, dim), slope, shared).reshape(-1)
    results = []
    for _ in range(2):                                                          # twice: the same bits
        DY = Guarded(n, off, init=dy)
        DX = DY if in_place else Guarded(n, off)
        base = f32(np.linspace(-1, 1, slope.size))
        DS = torch.from_numpy(base.copy()).cuda()
        capi.check(capi.lib().b2c_prelu_backward(N, Cc, dim, int(shared), Xin.ptr(), DY.ptr(), capi._p(S), DX.ptr(), capi._p(DS),
                                                 capi._p(ws), ws.numel(), None))
        dx = DX.read().copy()
        np.testing.assert_array_equal(dx, dx_f32)
        ds = DS.cpu().numpy() - base.astype(np.float64)                      # added into, not overwritten
        assert np.all(np.abs(ds - ds_ref) <= 4 * 2.0 ** -24 * (mag + np.abs(base)) + 1e-30), (ds, ds_ref)
        results.append(DS.cpu().numpy())
    assert np.array_equal(results[0].view(np.uint32), results[1].view(np.uint32))


@pytest.mark.parametrize("case", [0, 4, 5])
def test_prelu_backward_with_dx_or_dslope_null(case):
    shape = PRELU_SHAPES[case]
    N, Cc, dim = shape
    for shared in (False, True):
        x, slope, dy = prelu_case(shape, shared, 99)
        X, DY, S = (torch.from_numpy(a.reshape(-1)).cuda() for a in (x, dy, slope))
        ws = torch.zeros(max(1, capi.prelu_workspace_bytes(N, Cc, dim, shared)), dtype=torch.uint8, device="cuda")
        DS = torch.zeros_like(S)
        capi.prelu_backward(N, Cc, dim, shared, X, DY, S, None, DS, ws)             # slope gradient only
        DS_full = torch.zeros_like(S)
        DX = torch.full_like(X, float("nan"))
        capi.prelu_backward(N, Cc, dim, shared, X, DY, S, DX, DS_full, ws)
        assert torch.equal(DS, DS_full)
        DX2 = torch.full_like(X, float("nan"))
        capi.prelu_backward(N, Cc, dim, shared, X, DY, S, DX2, None, None)          # dx only: no workspace needed
        assert torch.equal(DX, DX2)
        capi.prelu_backward(N, Cc, dim, shared, X, DY, S, None, None, None)         # nothing to do
    if capi.prelu_workspace_bytes(N, Cc, dim, False):
        with pytest.raises(capi.B2CError, match="workspace too small"):
            capi.prelu_backward(N, Cc, dim, False, X, DY, torch.zeros(Cc, device="cuda"), None, torch.zeros(Cc, device="cuda"), None)


# ---- through TrainNet ------------------------------------------------------------------------------------------------------------
def rel(a, b):
    return float(np.abs(np.asarray(a, np.float64) - b).max() / max(np.abs(b).max(), 1e-30))


def init_params(H, W, classes, shared, seed):
    rng = np.random.default_rng(seed)
    out = []
    for i, sh in enumerate(no.net_param_shapes(H, W, classes, shared)):
        if i == 2:
            out.append(f32(rng.uniform(0.1, 0.4, sh if sh else (1,))))
        else:
            fan = int(np.prod(sh[1:])) if len(sh) > 1 else 1
            out.append(f32(rng.standard_normal(sh if sh else (1,)) * (0.5 / np.sqrt(fan))))
    return out


@pytest.mark.parametrize("shared", [False, True])
def test_neuron_net_through_trainnet(shared):
    """conv -> in-place PReLU -> conv -> ELU -> Power -> AbsVal -> BNLL -> Exp -> Log -> InnerProduct -> SoftmaxWithLoss, and a
    forward-only Threshold on the second conv: loss, blobs, every parameter gradient (the slope in both forms) and three SGD steps
    against the float64 oracle; one step with iter_size 2 equals one step on the double batch."""
    N, H, W, classes = 4, 6, 5, 3
    lr, mom = 0.05, 0.9
    solver = f'base_lr: {lr} lr_policy: "fixed" momentum: {mom} max_iter: 10'
    t = host_api.Trainer(no.net_prototxt(N, H, W, classes, shared), solver, num_classes=classes)
    assert np.array_equal(t.get_param(2, 0), np.full(1 if shared else 6, 0.3, np.float32))     # the filler's constant
    params = init_params(H, W, classes, shared, 5)
    for i, p in enumerate(params):
        t.set_param(i, p)
    rng = np.random.default_rng(6)
    x = f32(rng.standard_normal((N, 3, H, W)))
    lab = f32(rng.integers(0, classes, N))
    t.set_blob("data", x)
    t.set_blob("label", lab)
    loss = t.forward_backward()
    want, grads, blobs = no.net_forward_backward(params, x, lab)
    assert abs(loss - want) <= 1e-5 * abs(want), (loss, want)
    for nm, v in blobs.items():
        got = t.get_blob(nm).reshape(v.shape)
        if nm == "thr":
            c2 = t.get_blob("c2")
            assert np.array_equal(t.get_blob("thr"), (c2 > np.float32(0.3)).astype(np.float32))
        else:
            assert rel(got, v) < 1e-5, nm
    for i, g in enumerate(grads):
        assert rel(t.get_param(i, 1).reshape(g.shape), g) < 1e-4, i
    ws = [p.astype(np.float64) for p in params]
    hs = [np.zeros_like(w) for w in ws]
    for _ in range(3):
        _, gs, _ = no.net_forward_backward(ws, x, lab)
        for i in range(len(ws)):
            hs[i] = mom * hs[i] + lr * gs[i]
            ws[i] = ws[i] - hs[i]
    t.clear_param_diffs()
    t.step(3)
    for i, w in enumerate(ws):
        assert rel(t.get_param(i, 0).reshape(w.shape), w) < 1e-4, i
    # iter_size 2: the solver runs two micro-batches of N (the Input layer's resident batch both times), accumulates the diffs and
    # folds 1/iter_size into the update -- one SGD step on the 2N batch [x; x], as the oracle and a batch-2N trainer take it
    x2, lab2 = np.concatenate([x, x]), np.concatenate([lab, lab])
    _, g2, _ = no.net_forward_backward(params, x2, lab2)
    want = [p.astype(np.float64) - lr * g for p, g in zip(params, g2)]
    stepped = []
    for batch, extra, xs, ls in ((N, " iter_size: 2", x, lab), (2 * N, "", x2, lab2)):
        t2 = host_api.Trainer(no.net_prototxt(batch, H, W, classes, shared), solver + extra, num_classes=classes)
        for i, p in enumerate(params):
            t2.set_param(i, p)
        t2.set_blob("data", xs)
        t2.set_blob("label", ls)
        t2.clear_param_diffs()
        t2.step(1)
        stepped.append([t2.get_param(i, 0).reshape(w.shape).astype(np.float64) - params[i] for i, w in enumerate(want)])
    # the updates (new - old weights) against float64, and iter_size 2 against batch 2N; the new weights are float32, so each update
    # is known to within one ulp of the weight on top of the relative bound
    for i, w in enumerate(want):
        d = w - params[i]
        ulp = np.spacing(np.maximum(np.abs(params[i]), np.abs(w)).astype(np.float32)).astype(np.float64)
        tol = 1e-4 * np.abs(d).max()
        assert np.all(np.abs(stepped[0][i] - d) <= tol + ulp), i
        assert np.all(np.abs(stepped[0][i] - stepped[1][i]) <= tol + 2 * ulp), i


def test_out_of_place_prelu_keeps_no_copy_and_matches_in_place():
    N, H, W, classes = 2, 4, 4, 3
    solver = 'base_lr: 0.05 lr_policy: "fixed" max_iter: 10'
    params = init_params(H, W, classes, False, 8)
    rng = np.random.default_rng(9)
    x, lab = f32(rng.standard_normal((N, 3, H, W))), f32(rng.integers(0, classes, N))
    outs = []
    for in_place in (True, False):
        t = host_api.Trainer(no.net_prototxt(N, H, W, classes, False, prelu_in_place=in_place), solver, num_classes=classes)
        for i, p in enumerate(params):
            t.set_param(i, p)
        t.set_blob("data", x)
        t.set_blob("label", lab)
        outs.append((t.forward_backward(), [t.get_param(i, 1) for i in range(len(params))]))
    assert outs[0][0] == outs[1][0]
    for a, b in zip(outs[0][1], outs[1][1]):
        assert np.array_equal(a, b)


def test_prelu_misaligned_call_fits_the_reported_workspace():
    """a channel-shared 32 x 64 x 32 x 32 PReLU 4 bytes off takes the scalar path with the workspace the query reported, twice on
    the same (once-zeroed) workspace, with the same bits"""
    N, Cc, dim = 32, 64, 32 * 32
    x, slope, dy = prelu_case((N, Cc, dim), True, 21)
    ws = torch.zeros(capi.prelu_workspace_bytes(N, Cc, dim, True), dtype=torch.uint8, device="cuda")
    assert ws.numel() > 0
    X, DY = Guarded(x.size, 1, init=x), Guarded(x.size, 1, init=dy)
    S = torch.from_numpy(slope).cuda()
    assert not capi.neuron_plan("prelu_backward", N, Cc, dim, shared=True, ptrs=(X.ptr().value, DY.ptr().value))["vec"]
    _, ds_ref, mag = no.prelu_backward(x, dy, slope, True)
    got = []
    for _ in range(2):
        DS = torch.zeros(1, device="cuda")
        capi.check(capi.lib().b2c_prelu_backward(N, Cc, dim, 1, X.ptr(), DY.ptr(), capi._p(S), None, capi._p(DS), capi._p(ws), ws.numel(),
                                                 None))
        got.append(DS.cpu().numpy())
    assert np.array_equal(got[0].view(np.uint32), got[1].view(np.uint32))
    assert abs(float(got[0][0]) - ds_ref[0]) <= 4 * 2.0 ** -24 * mag[0]

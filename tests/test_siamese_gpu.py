"""ContrastiveLoss kernels per element against the float64 forms of tests/siamese_oracle.py, Slice in a net, and the weight-sharing
semantics of the reference's test_net.cpp (SharedWeightsDataNet / DiffNet / Update / Resume) through TrainNet, then a siamese net
on conv layers against the oracle: loss, every owner's gradient and three SGD steps.

Bounds: dist_sq[n] is float(sum_c float(d^2)) with the channel sum in double (b2c.h), d = a - b rounded once, so |dist_sq - d2| <=
4 * 2^-24 * d2 (the rounding of d, of d^2 and of the final float); the loss sums float terms in double, each term within a few
roundings of its float64 value."""
import ctypes

import numpy as np
import pytest

import siamese_oracle as so
from cases import Guarded

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import caffe_mpi_b200 as m  # noqa: E402
from caffe_mpi_b200 import capi, host_api  # noqa: E402

U = 2.0 ** -24


def st():
    return capi._stream()


def bits(a):
    return np.ascontiguousarray(a).view(np.int32)


def within(got, ref, bound, what):
    err = np.abs(got.astype(np.float64) - ref)
    bad = np.flatnonzero(~(err <= bound))
    assert bad.size == 0, f"{what}: {bad.size} out of bound, first {bad[:5]}: got {got.reshape(-1)[bad[:3]]} ref {ref.reshape(-1)[bad[:3]]}"


def rel(a, ref, floor=1e-20):
    return float(np.max(np.abs(a.reshape(-1) - ref.reshape(-1))) / max(np.max(np.abs(ref)), floor))


# ------------------------------------------------------------------------------------------------------------ ContrastiveLoss kernels
# 10^5 x 4096 (1.6 GB per operand) is test_contrastive_large below: there the oracle runs on the device, in float64 and in chunks,
# instead of in host numpy with its temporaries
SIZES = [(N, C) for N in (1, 64, 512) for C in (1, 2, 3, 128, 4096)] + [(100000, C) for C in (1, 2, 3, 128)]


@pytest.mark.parametrize("N,C", SIZES, ids=[f"{n}x{c}" for n, c in SIZES])
@pytest.mark.parametrize("legacy", [0, 1], ids=["new", "legacy"])
@pytest.mark.parametrize("off", [0, 1], ids=["aligned", "off4"])
def test_contrastive_per_element(N, C, legacy, off):
    rng = np.random.default_rng(N * 31 + C + legacy)
    scale = 1.0 / np.sqrt(C)              # keeps distances near the margin so both branches run
    a = (rng.uniform(-1, 1, (N, C)) * scale).astype(np.float32)
    b = (rng.uniform(-1, 1, (N, C)) * scale).astype(np.float32)
    y = rng.choice(np.array([0.0, 1.0, 0.7, -1.0, 1.3], np.float32), N)
    margin = 0.8 if not legacy else 0.5
    L = m.lib()
    runs = []
    for _ in range(2):
        A, B, Y = Guarded(a.size, off, a), Guarded(b.size, off, b), Guarded(N, off, y)
        D, D2, LOSS = Guarded(a.size, off), Guarded(N, off), Guarded(1, off)
        capi.check(L.b2c_contrastive_loss_forward(N, C, A.ptr(), B.ptr(), Y.ptr(), margin, legacy, D.ptr(), D2.ptr(), LOSS.ptr(), st()))
        diff, d2, loss = D.read().reshape(N, C).copy(), D2.read().copy(), LOSS.read().copy()
        DA, DB, DA1 = Guarded(a.size, off), Guarded(a.size, off), Guarded(a.size, off)
        DD, DD2 = Guarded(a.size, off, diff), Guarded(N, off, d2)
        alpha = 0.75 / N
        capi.check(L.b2c_contrastive_loss_backward(N, C, DD.ptr(), DD2.ptr(), Y.ptr(), margin, legacy, alpha, DA.ptr(), DB.ptr(), st()))
        capi.check(L.b2c_contrastive_loss_backward(N, C, DD.ptr(), DD2.ptr(), Y.ptr(), margin, legacy, alpha, DA1.ptr(), None, st()))
        da, db, da1 = (G.read().reshape(N, C).copy() for G in (DA, DB, DA1))
        runs.append((diff, d2, loss, da, db))
    for x, x2 in zip(runs[0], runs[1]):
        assert np.array_equal(bits(x), bits(x2)), "a repeat call changed the bits"
    diff, d2, loss, da, db = runs[0]
    assert np.array_equal(bits(da1), bits(da)), "db = null changed da"
    nz = da != 0                            # db = -da bit for bit; a 0 is +0 where the hinge zeroed the pair, else -da's sign
    assert np.array_equal(bits(db[nz]), bits(-da[nz])) and np.all(db[~nz] == 0), "db is not -da"
    a64, b64 = a.astype(np.float64), b.astype(np.float64)
    ref_loss, ref_diff, ref_d2 = so.contrastive_forward(a64, b64, y, margin, bool(legacy))
    within(diff, ref_diff, U * np.abs(ref_diff), "diff")
    within(d2, ref_d2, 4 * U * ref_d2 + 1e-45, "dist_sq")
    # each term from dist_sq (4u relative): similar 4u d2; legacy u (5 d2 + margin) (the subtraction's rounding); otherwise
    # m = margin - sqrtf(d2) is within E = u (4 d + margin) and m^2 within E (2 m + E) + u m^2.  The loss: the terms' bounds / 2N
    # plus the float rounding of the sum and of / N.  Everything doubled for slack.
    d = np.sqrt(ref_d2)
    sim = so.similar(y)
    if legacy:
        dis_err = U * (5 * ref_d2 + margin)
    else:
        E = U * (4 * d + margin)
        mh = np.maximum(margin - d, 0)
        dis_err = E * (2 * mh + E) + U * mh * mh
    term_err = np.where(sim, 4 * U * ref_d2, dis_err)
    within(np.array([loss[0]]), np.array([ref_loss]), 2 * (term_err.sum() / N / 2 + 2 * U * abs(ref_loss)) + 1e-45, "loss")
    # backward on the kernel's own diff / dist_sq (the hinge and the 1e-4 decided on the float dist_sq)
    d2f = d2.astype(np.float64)
    ref_da, _ = so.contrastive_backward(diff.astype(np.float64), d2f, y, margin, bool(legacy), loss_weight=0.75)
    # a few roundings relative (alpha, sqrtf, the division, the product), plus margin - sqrtf(d2)'s rounding, which is relative to
    # margin + d rather than to the (possibly tiny) difference
    df = np.sqrt(d2f)
    hinge_err = np.where(so.similar(y) | bool(legacy), 0.0, 4 * U * (0.75 / N) * (margin + df) / (df + 1e-4))
    within(da, ref_da, 8 * U * np.abs(ref_da) + hinge_err[:, None] * np.abs(diff) + 1e-45, "da")


@pytest.mark.parametrize("legacy", [0, 1], ids=["new", "legacy"])
def test_contrastive_large(legacy):
    """N = 10^5 pairs of C = 4096 channels: an 8-CTA cluster with every warp looping over 4096 channels for ~780 pairs.  Inputs are
    drawn and checked on the device: diff against torch's float32 subtraction (the same single rounding), dist_sq, the loss and
    da against float64 sums taken 2 000 pairs at a time, under the per-element bounds of test_contrastive_per_element."""
    N, C = 100000, 4096
    g = torch.Generator(device="cuda").manual_seed(3 + legacy)
    a = (torch.rand(N, C, device="cuda", generator=g) * 2 - 1) / 64
    b = (torch.rand(N, C, device="cuda", generator=g) * 2 - 1) / 64
    y = (torch.rand(N, device="cuda", generator=g) < 0.5).float()
    margin = 0.8 if not legacy else 0.5
    diff, d2, loss = torch.empty_like(a), torch.empty(N, device="cuda"), torch.empty(1, device="cuda")
    da, db = torch.empty_like(a), torch.empty_like(a)
    L = m.lib()
    ptr = lambda t: ctypes.c_void_p(t.data_ptr())
    torch.cuda.synchronize()                  # the inputs were drawn on torch's stream
    capi.check(L.b2c_contrastive_loss_forward(N, C, ptr(a), ptr(b), ptr(y), margin, legacy, ptr(diff), ptr(d2), ptr(loss), st()))
    loss1, d2_1 = loss.clone(), d2.clone()
    capi.check(L.b2c_contrastive_loss_forward(N, C, ptr(a), ptr(b), ptr(y), margin, legacy, ptr(diff), ptr(d2), ptr(loss), st()))
    alpha = 1.0 / N
    capi.check(L.b2c_contrastive_loss_backward(N, C, ptr(diff), ptr(d2), ptr(y), margin, legacy, alpha, ptr(da), ptr(db), st()))
    torch.cuda.synchronize()
    assert torch.equal(loss1.view(torch.int32), loss.view(torch.int32)) and torch.equal(d2_1.view(torch.int32), d2.view(torch.int32))
    total, term_err = 0.0, 0.0
    for lo in range(0, N, 2000):
        sl = slice(lo, lo + 2000)
        assert torch.equal(diff[sl], a[sl] - b[sl])
        ref_diff = a[sl].double() - b[sl].double()
        ref_d2 = (ref_diff * ref_diff).sum(dim=1)
        assert bool(((d2[sl].double() - ref_d2).abs() <= 4 * U * ref_d2 + 1e-45).all()), lo
        d = ref_d2.sqrt()
        sim = y[sl] != 0
        if legacy:
            dis, dis_err = (margin - ref_d2).clamp(min=0), U * (5 * ref_d2 + margin)
        else:
            mh = (margin - d).clamp(min=0)
            E = U * (4 * d + margin)
            dis, dis_err = mh * mh, E * (2 * mh + E) + U * mh * mh
        total += float(torch.where(sim, ref_d2, dis).sum())
        term_err += float(torch.where(sim, 4 * U * ref_d2, dis_err).sum())
        # backward on the kernel's own diff / dist_sq
        d2f, df = d2[sl].double(), d2[sl].double().sqrt()
        if legacy:
            coef = torch.where(margin - d2f > 0, -alpha, 0.0)
        else:
            coef = torch.where(margin - df > 0, -alpha * (margin - df) / (df + 1e-4), 0.0)
        coef = torch.where(sim, torch.full_like(coef, alpha), coef)
        ref_da = coef[:, None] * diff[sl].double()
        herr = torch.where(sim | bool(legacy), 0.0, 4 * U * alpha * (margin + df) / (df + 1e-4))
        assert bool(((da[sl].double() - ref_da).abs() <= 8 * U * ref_da.abs() + herr[:, None] * diff[sl].double().abs() + 1e-45).all()), lo
        nz = da[sl] != 0
        assert torch.equal(db[sl][nz], -da[sl][nz]) and bool((db[sl][~nz] == 0).all())
    ref_loss = total / N / 2
    assert abs(float(loss[0]) - ref_loss) <= 2 * (term_err / N / 2 + 2 * U * abs(ref_loss)), (float(loss[0]), ref_loss)


def test_contrastive_rejects_bad_arguments():
    L = m.lib()
    X = Guarded(8)
    assert L.b2c_contrastive_loss_forward(0, 2, X.ptr(), X.ptr(), X.ptr(), 1.0, 0, X.ptr(), X.ptr(), X.ptr(), st()) != 0
    assert L.b2c_contrastive_loss_forward(2, 0, X.ptr(), X.ptr(), X.ptr(), 1.0, 0, X.ptr(), X.ptr(), X.ptr(), st()) != 0
    assert L.b2c_contrastive_loss_forward(2, 2, None, X.ptr(), X.ptr(), 1.0, 0, X.ptr(), X.ptr(), X.ptr(), st()) != 0
    assert L.b2c_contrastive_loss_backward(2, 2, X.ptr(), X.ptr(), X.ptr(), 1.0, 0, 1.0, None, None, st()) != 0
    assert L.b2c_contrastive_loss_backward(-1, 2, X.ptr(), X.ptr(), X.ptr(), 1.0, 0, 1.0, X.ptr(), None, st()) != 0


# ------------------------------------------------------------------------------------------------------------ Slice in a net
@pytest.mark.parametrize("axis,param", [(0, "axis: 0 slice_point: 1"), (1, "slice_dim: 1 slice_point: 2"), (3, "axis: -1 slice_point: 3")])
def test_slice_forward_backward(axis, param):
    """x -> Slice -> (t0, t1); only t0 feeds the loss (EuclideanLoss against a target), so t1's diff is never written: the bottom's
    diff is the loss gradient in t0's window and zero in t1's.  force_backward makes the Input's diff reachable."""
    shape = (3, 5, 2, 4)
    rng = np.random.default_rng(axis)
    x = rng.standard_normal(shape).astype(np.float32)
    parts = so.slice_forward(x, axis, [int(param.split()[-1])])
    tgt = rng.standard_normal(parts[0].shape).astype(np.float32)
    net = ('name: "s" force_backward: true\n'
           'layer { name: "in" type: "Input" top: "x" top: "t" input_param { shape { %s } shape { %s } } }\n'
           'layer { name: "slice" type: "Slice" bottom: "x" top: "t0" top: "t1" slice_param { %s } }\n'
           'layer { name: "loss" type: "EuclideanLoss" bottom: "t0" bottom: "t" top: "loss" }\n'
           % (" ".join("dim: %d" % d for d in shape), " ".join("dim: %d" % d for d in tgt.shape), param))
    t = host_api.Trainer(net, 'base_lr: 0.01 lr_policy: "fixed" max_iter: 1', num_classes=2)
    t.set_blob("x", x)
    t.set_blob("t", tgt)
    t.forward_backward()
    assert np.array_equal(t.get_blob("t0"), parts[0].reshape(-1)) and np.array_equal(t.get_blob("t1"), parts[1].reshape(-1))
    g0 = (parts[0].astype(np.float64) - tgt) / parts[0].shape[0]
    ref = so.slice_backward([t.get_blob("t0", diff=True).reshape(parts[0].shape), np.zeros_like(parts[1])], axis)
    assert np.array_equal(t.get_blob("x", diff=True), ref.reshape(-1))
    assert rel(t.get_blob("t0", diff=True), g0) <= 1e-6


# ------------------------------------------------------------------------------------------------------------ test_net.cpp sharing
def _shared_ips(share=True, target="y2"):
    """test_net.cpp's SharedWeights nets: x -> ip1, ip2 (no bias, one weight when shared) -> EuclideanLoss(y1, y2)"""
    p = 'param { name: "sharedweights" } ' if share else ""
    return ('name: "SharedWeightsNetwork" force_backward: true\n'
            'layer { name: "data" type: "Input" top: "data" input_param { shape { dim: 10 dim: 10 } } }\n'
            'layer { name: "innerproduct1" type: "InnerProduct" bottom: "data" top: "innerproduct1" %s'
            'inner_product_param { num_output: 10 bias_term: false weight_filler { type: "gaussian" std: 10 } } }\n'
            'layer { name: "innerproduct2" type: "InnerProduct" bottom: "data" top: "innerproduct2" %s'
            'inner_product_param { num_output: 10 bias_term: false weight_filler { type: "gaussian" std: 10 } } }\n'
            'layer { name: "loss" type: "EuclideanLoss" bottom: "innerproduct1" bottom: "innerproduct2" top: "loss" }\n' % (p, p))


SGD = 'base_lr: 1 lr_policy: "fixed" max_iter: 10'


def test_shared_weights_data_net():
    """SharedWeightsDataNet: two InnerProducts on one input with one weight -- the loss between them is 0"""
    t = host_api.Trainer(_shared_ips(), SGD, num_classes=2)
    assert t.num_params() == 1 and t.num_learnable() == 1
    assert t.forward_backward() == 0.0
    assert np.array_equal(t.get_blob("innerproduct1"), t.get_blob("innerproduct2"))


def test_shared_weights_diff_net():
    """SharedWeightsDiffNet: the two uses' gradients cancel -- the shared diff is 0"""
    t = host_api.Trainer(_shared_ips(), SGD, num_classes=2)
    t.forward_backward()
    assert np.all(t.get_param(0, 1) == 0.0)


def test_shared_weights_update():
    """SharedWeightsUpdate: the two layers hold distinct Blob objects over one data and one diff storage; the shared diff is the
    sum of the unshared net's two diffs; one SGD step (lr 1) gives data - diff"""
    rng = np.random.default_rng(5)
    x = rng.standard_normal((10, 10)).astype(np.float32)
    w = rng.standard_normal((10, 10)).astype(np.float32)
    w2 = rng.standard_normal((10, 10)).astype(np.float32)
    sh = host_api.Trainer(_shared_ips(), SGD, num_classes=2)
    ip1, ip2 = [[nm for nm, _ in sh.layers()].index(n) for n in ("innerproduct1", "innerproduct2")]
    o1, d1, g1 = sh.layer_blob_pointers(ip1, 0)
    o2, d2, g2 = sh.layer_blob_pointers(ip2, 0)
    assert o1 != o2 and d1 == d2 and g1 == g2
    un = host_api.Trainer(_shared_ips(share=False), SGD, num_classes=2)
    u1, u2 = un.layer_blob_pointers(ip1, 0), un.layer_blob_pointers(ip2, 0)
    assert u1[1] != u2[1] and u1[2] != u2[2]
    # a net where the two uses do not cancel: ip2 reads a second input through its own (shared) weight
    net = _shared_ips().replace('bottom: "data" top: "innerproduct2"', 'bottom: "data2" top: "innerproduct2"').replace(
        'layer { name: "innerproduct1"', 'layer { name: "data2" type: "Input" top: "data2" input_param { shape { dim: 10 dim: 10 } } }\n'
        'layer { name: "innerproduct1"')
    sh = host_api.Trainer(net, SGD, num_classes=2)
    un = host_api.Trainer(net.replace('param { name: "sharedweights" } ', ""), SGD, num_classes=2)
    for t in (sh, un):
        t.set_blob("data", x)
        t.set_blob("data2", w2)
    sh.set_param(0, w)
    un.set_param(0, w); un.set_param(1, w)
    sh.forward_backward(); un.forward_backward()
    shared = sh.get_param(0, 1)
    assert np.abs(shared).max() > 0
    np.testing.assert_allclose(shared, un.get_param(0, 1) + un.get_param(1, 1), rtol=1e-6, atol=1e-6 * np.abs(shared).max())
    sh.clear_param_diffs()
    sh.step(1)
    np.testing.assert_allclose(sh.get_param(0, 0), w.reshape(-1) - shared, rtol=1e-6, atol=1e-6 * np.abs(shared).max())
    # both layers read the one updated storage: their tops agree with the host product on the new weights
    sh.forward_backward()
    wn = sh.get_param(0, 0).reshape(10, 10).astype(np.float64)
    np.testing.assert_allclose(sh.get_blob("innerproduct1"), (x @ wn.T).reshape(-1), rtol=1e-4, atol=1e-3)
    np.testing.assert_allclose(sh.get_blob("innerproduct2"), (w2 @ wn.T).reshape(-1), rtol=1e-4, atol=1e-3)


def test_shared_weights_resume(tmp_path):
    """SharedWeightsResume: step, snapshot, restore into a fresh net; the two layers read one storage and the next step is bitwise
    the uninterrupted run's"""
    net = so.siamese_prototxt(N=6)
    solver = 'base_lr: 0.01 lr_policy: "fixed" momentum: 0.9 max_iter: 100'
    rng = np.random.default_rng(9)
    pair = rng.uniform(0, 1, (6, 2, 12, 12)).astype(np.float32)
    sim = np.array([1, 0, 1, 0, 0, 1], np.float32)

    def make():
        t = host_api.Trainer(net, solver, num_classes=2)
        t.set_blob("pair_data", pair)
        t.set_blob("sim", sim)
        return t
    a = make()
    assert a.num_learnable() == 6
    a.step(2)
    state = a.snapshot(str(tmp_path / "siam"))
    a.step(1)
    b = make()
    b.restore(state)
    assert b.iter() == 2
    b.step(1)
    for i in range(6):
        assert np.array_equal(bits(a.get_param(i, 0)), bits(b.get_param(i, 0))), i
        assert np.array_equal(bits(a.get_param(i, 2)), bits(b.get_param(i, 2))), i
    assert a.forward_backward() == b.forward_backward()
    assert np.array_equal(bits(a.get_blob("feat_p")), bits(b.get_blob("feat_p")))
    # the _p tower reads the owners' storage: the same half through it gives the same features
    b.set_blob("pair_data", np.concatenate([pair[:, :1], pair[:, :1]], axis=1))
    b.forward_backward()
    assert np.array_equal(b.get_blob("feat"), b.get_blob("feat_p"))


# ------------------------------------------------------------------------------------------------------------ siamese net vs oracle
def _siamese(legacy, rng, N=8):
    shapes = so.siamese_param_shapes()
    t = host_api.Trainer(so.siamese_prototxt(N=N, legacy=legacy), 'base_lr: 0.05 lr_policy: "fixed" momentum: 0.9 max_iter: 100',
                         num_classes=2)
    params = []
    for i, shp in enumerate(shapes):
        fan = int(np.prod(shp[1:])) if len(shp) > 1 else 1
        p = (rng.standard_normal(shp) / np.sqrt(fan)).astype(np.float32) if len(shp) > 1 else rng.uniform(-0.1, 0.1, shp).astype(np.float32)
        t.set_param(i, p)
        params.append(p)
    pair = rng.uniform(0, 1, (N, 2, 12, 12)).astype(np.float32)
    sim = (rng.uniform(0, 1, N) < 0.5).astype(np.float32)
    t.set_blob("pair_data", pair)
    t.set_blob("sim", sim)
    return t, params, pair, sim


@pytest.mark.parametrize("legacy", [False, True], ids=["new", "legacy"])
def test_siamese_net_matches_oracle(legacy):
    t, params, pair, sim = _siamese(legacy, np.random.default_rng(17 + legacy))
    assert t.num_params() == 6
    loss = t.forward_backward()
    ref_loss, grads, (fa, fb) = so.siamese_forward_backward(params, pair, sim, legacy=legacy)
    assert abs(loss - ref_loss) <= 1e-4 * abs(ref_loss), (loss, ref_loss)
    assert rel(t.get_blob("feat"), fa) <= 1e-4 and rel(t.get_blob("feat_p"), fb) <= 1e-4
    for i, g in enumerate(grads):           # the owners' gradients: the sum over both towers (1e-3 behind several layers)
        assert rel(t.get_param(i, 1), g) <= (1e-4 if i >= 4 else 1e-3), i


def test_siamese_net_sgd_steps_match_oracle():
    t, params, pair, sim = _siamese(False, np.random.default_rng(23))
    ref = [p.astype(np.float64) for p in params]
    hist = [np.zeros_like(p) for p in ref]
    losses, ref_losses = [], []
    lr_mult = [1, 2, 1, 2, 1, 2]
    for _ in range(3):
        loss, grads, _ = so.siamese_forward_backward(ref, pair, sim)
        ref_losses.append(loss)
        for i, g in enumerate(grads):       # SGD with momentum 0.9, no weight decay (sgd_solver.cpp ComputeUpdateValue)
            hist[i] = 0.9 * hist[i] + 0.05 * lr_mult[i] * g
            ref[i] = ref[i] - hist[i]
        t.step(1)
        losses.append(t.loss())
    np.testing.assert_allclose(losses, ref_losses, rtol=1e-4)
    for i in range(6):
        assert rel(t.get_param(i, 0), ref[i]) <= 1e-4, i


# ------------------------------------------------------------------------------------------------------------ shared wgrad routes
# (N, C, H, W, O, k, pad): a shared weight on each weight-gradient regime a conv layer can take; test_shared_wgrad_routes_are_covered
# checks that the set reaches a split-K plan and the pre-split staged path
WGRAD = [(32, 16, 56, 56, 16, 3, 1), (8, 64, 14, 14, 64, 3, 1), (4, 32, 28, 28, 32, 3, 1), (16, 256, 14, 14, 64, 1, 0), (2, 3, 9, 9, 5, 3, 0)]


def _plan(c):
    N, C, H, W, O, k, p = c
    return m.ConvDesc(capi.ConvParams.make(N, C, H, W, O, k, 1, p)).wgrad_plan()


def test_shared_wgrad_routes_are_covered():
    plans = [_plan(c) for c in WGRAD]
    assert any(p["splits"] > 1 for p in plans), plans
    assert any(p["presplit_dy"] for p in plans), plans
    assert len({p["route"] for p in plans}) >= 3, plans


@pytest.mark.parametrize("c", WGRAD, ids=["x".join(map(str, c)) for c in WGRAD])
def test_shared_weight_gradient_sums_on_every_wgrad_route(c):
    """Two conv layers that share weight and bias by name, on two inputs, EuclideanLoss between them: the owner's diff equals the
    sum of the unshared net's two diffs on the same weights and inputs (the second use ADDS into the first's dW on this route)."""
    N, C, H, W, O, k, p = c
    plan = _plan(c)
    rng = np.random.default_rng(sum(c))

    def net(share):
        ps = 'param { name: "w" } param { name: "b" } ' if share else ""
        conv = ('layer { name: "%s" type: "Convolution" bottom: "%s" top: "%s" ' + ps +
                'convolution_param { num_output: %d kernel_size: %d pad: %d } }\n')
        return ('name: "wg" force_backward: true\nlayer { name: "in" type: "Input" top: "x1" top: "x2" input_param { shape { dim: %d dim: %d '
                'dim: %d dim: %d } shape { dim: %d dim: %d dim: %d dim: %d } } }\n' % (N, C, H, W, N, C, H, W) +
                conv % ("ca", "x1", "ya", O, k, p) + conv % ("cb", "x2", "yb", O, k, p) +
                'layer { name: "loss" type: "EuclideanLoss" bottom: "ya" bottom: "yb" top: "loss" }\n')
    w = (rng.standard_normal((O, C, k, k)) / np.sqrt(C * k * k)).astype(np.float32)
    bias = rng.uniform(-0.1, 0.1, O).astype(np.float32)
    x1, x2 = (rng.standard_normal((N, C, H, W)).astype(np.float32) for _ in range(2))
    sh = host_api.Trainer(net(True), SGD, num_classes=2)
    un = host_api.Trainer(net(False), SGD, num_classes=2)
    assert sh.num_params() == 2 and un.num_params() == 4
    sh.set_param(0, w); sh.set_param(1, bias)
    for i, v in enumerate((w, bias, w, bias)):
        un.set_param(i, v)
    for t in (sh, un):
        t.set_blob("x1", x1)
        t.set_blob("x2", x2)
        t.forward_backward()
    # (the bias: ya and yb get opposite gradients, so its two uses cancel -- the sum is 0 up to rounding, at the scale of one use)
    for j in range(2):
        one_use = un.get_param(j, 1).astype(np.float64)
        got, ref = sh.get_param(j, 1).astype(np.float64), one_use + un.get_param(j + 2, 1)
        assert np.abs(one_use).max() > 0 and (j == 1 or np.abs(ref).max() > 0)
        assert np.abs(got - ref).max() <= 1e-5 * max(np.abs(ref).max(), np.abs(one_use).max() if j == 1 else 0.0), (plan, j)

"""Weight sharing through TrainNet's host logic on the stream-order model (tests/sim: fake CUDA runtime, host stand-ins for conv,
pooling, InnerProduct, SoftmaxWithLoss and cudaMemcpy2DAsync).  A siamese-shaped net -- Slice -> two conv towers whose every blob is
shared by name -> Concat -> InnerProduct -> SoftmaxWithLoss -- with one reduce bucket per parameter, so an owner released before
a sharer's backward has added into its diff, or a sharer releasing into the scheduler, shows up as a wrong update:
- three SGD steps against a float64 oracle with tied weights (the gradient of a tied weight is the sum over its uses) under the
  four extreme stream orders;
- iter_size 2 on a resident batch equals iter_size 1;
- two in-process ranks through P2PSync end with the same bits and equal one solver on the whole batch."""
import ctypes as C

import numpy as np
import pytest

from test_trainer_sim import STEP_MODES, _set_modes, sim_host  # noqa: F401  (sim_host: the module fixture)

torch = pytest.importorskip("torch")

SOLVER = 'base_lr: 0.05 lr_policy: "fixed" momentum: 0.9 weight_decay: 0.0005 max_iter: 100'
H, CONV, FEAT, CLS = 8, 3, 4, 5


def net(N, share=True):
    def p(nm):
        return 'param { name: "%s" } ' % nm if share else ""
    s = ('name: "siamese_sim" reduce_buckets: 100\n'
         'layer { name: "pair" type: "Input" top: "pair_data" top: "label" input_param { shape { dim: %d dim: 2 dim: %d dim: %d } '
         'shape { dim: %d } } }\n' % (N, H, H, N))
    s += 'layer { name: "slice" type: "Slice" bottom: "pair_data" top: "a" top: "b" slice_param { axis: 1 } }\n'
    for x in ("a", "b"):
        s += ('layer { name: "conv_%s" type: "Convolution" bottom: "%s" top: "conv_%s" %s%s convolution_param { num_output: %d '
              'kernel_size: 3 } }\n' % (x, x, x, p("cw"), p("cb"), CONV))
        s += 'layer { name: "pool_%s" type: "Pooling" bottom: "conv_%s" top: "pool_%s" pooling_param { pool: MAX kernel_size: 2 stride: 2 } }\n' % (x, x, x)
        s += ('layer { name: "feat_%s" type: "InnerProduct" bottom: "pool_%s" top: "feat_%s" %s%s inner_product_param { num_output: %d } }\n'
              % (x, x, x, p("fw"), p("fb"), FEAT))
    s += 'layer { name: "cat" type: "Concat" bottom: "feat_a" bottom: "feat_b" top: "cat" }\n'
    s += 'layer { name: "cls" type: "InnerProduct" bottom: "cat" top: "cls" inner_product_param { num_output: %d } }\n' % CLS
    s += 'layer { name: "loss" type: "SoftmaxWithLoss" bottom: "cls" bottom: "label" top: "loss" }\n'
    return s


P = (H - 2) // 2
SHAPES = [(CONV, 1, 3, 3), (CONV,), (FEAT, CONV * P * P), (FEAT,), (CLS, 2 * FEAT), (CLS,)]


def case(N, seed=3):
    rng = np.random.default_rng(seed)
    params = [(rng.standard_normal(s) / np.sqrt(np.prod(s[1:]))).astype(np.float32) if len(s) > 1 else
              rng.uniform(-0.1, 0.1, s).astype(np.float32) for s in SHAPES]
    data = rng.uniform(0, 1, (N, 2, H, H)).astype(np.float32)
    label = rng.integers(0, CLS, N).astype(np.float32)
    return params, data, label


def oracle_steps(params, data, label, steps, lr=0.05, mom=0.9, wd=0.0005):
    """float64 replay: the towers share every tensor, so autograd sums each tied gradient over both uses; SGD with momentum and L2
    decay as sgd_solver.cpp (history = mom * history + lr * (g + wd * w); w -= history)"""
    import torch.nn.functional as F
    w = [torch.tensor(p.astype(np.float64)) for p in params]
    h = [torch.zeros_like(t) for t in w]
    x = torch.tensor(data.astype(np.float64))
    y = torch.tensor(label.astype(np.int64))
    losses = []
    for _ in range(steps):
        P_ = [t.clone().requires_grad_(True) for t in w]

        def tower(v):
            v = F.max_pool2d(F.conv2d(v, P_[0], P_[1]), 2, 2)
            return F.linear(v.reshape(v.shape[0], -1), P_[2], P_[3])
        logits = F.linear(torch.cat([tower(x[:, 0:1]), tower(x[:, 1:2])], dim=1), P_[4], P_[5])
        loss = F.cross_entropy(logits, y)
        loss.backward()
        losses.append(float(loss.detach()))
        for i in range(len(w)):
            h[i] = mom * h[i] + lr * (P_[i].grad + wd * w[i])
            w[i] = w[i] - h[i]
    return losses, [t.numpy() for t in w], [t.numpy() for t in h]


def rel(a, ref, floor=1e-20):
    return float(np.max(np.abs(a.reshape(-1) - ref.reshape(-1))) / max(np.max(np.abs(ref)), floor))


def trainer(host, N, params, data, label, solver=SOLVER, share=True):
    t = host.Trainer(net(N, share), solver, num_classes=CLS)
    for i, p in enumerate(params):
        t.set_param(i, p)
    t.set_blob("pair_data", data)
    t.set_blob("label", label)
    return t


def test_siamese_sim_net_shares_by_name(sim_host):
    L = sim_host.lib()
    L.fakecuda_set_all_eager.argtypes = [C.c_int]
    L.fakecuda_set_all_eager(0)
    params, data, label = case(4)
    t = trainer(sim_host, 4, params, data, label)
    assert t.num_params() == 6 and t.num_learnable() == 6
    assert sim_host.Trainer(net(4, share=False), SOLVER, num_classes=CLS).num_params() == 10


@pytest.mark.parametrize("mode", sorted(STEP_MODES))
def test_siamese_sgd_steps_under_extreme_stream_orders(sim_host, mode):
    L = sim_host.lib()
    L.fakecuda_set_all_eager.argtypes = [C.c_int]
    L.fakecuda_set_all_eager(0)
    params, data, label = case(6)
    t = trainer(sim_host, 6, params, data, label)
    _set_modes(L, mode)
    try:
        ref_losses, ref_params, ref_hist = oracle_steps(params, data, label, 3)
        losses = []
        for k in range(3):
            t.step(1)
            losses.append(t.loss())
    finally:
        L.fakecuda_set_all_eager(0)
    np.testing.assert_allclose(losses, ref_losses, rtol=2e-4)
    for i in range(6):
        assert rel(t.get_param(i, 0), ref_params[i]) <= 2e-4, (mode, i)
        assert rel(t.get_param(i, 2), ref_hist[i], 1e-3 * np.abs(ref_hist[i]).max()) <= 5e-4, (mode, i)
        assert not t.get_param(i, 1).any(), (mode, i)


def test_siamese_iter_size_two_equals_one_pass(sim_host):
    L = sim_host.lib()
    L.fakecuda_set_all_eager.argtypes = [C.c_int]
    L.fakecuda_set_all_eager(0)
    params, data, label = case(6, seed=8)
    out = []
    for iter_size in (1, 2):
        t = trainer(sim_host, 6, params, data, label, SOLVER + " iter_size: %d" % iter_size)
        t.step(3)
        out.append(([t.get_param(i, 0) for i in range(6)], [t.get_param(i, 2) for i in range(6)], t.loss()))
    (p1, h1, l1), (p2, h2, l2) = out
    assert abs(l1 - l2) <= 1e-5 * abs(l1)
    for i in range(6):
        assert rel(p2[i], p1[i]) <= 1e-5 and rel(h2[i], h1[i], 1e-6) <= 1e-4, i


@pytest.mark.parametrize("mode", ["all-lazy", "all-eager"])
def test_siamese_two_ranks_equal_one_solver(sim_host, mode):
    L = sim_host.lib()
    L.sim_use_rank_stream.argtypes = [C.c_int]
    L.fakecuda_set_all_eager.argtypes = [C.c_int]
    L.sim_set_solver_count.argtypes = [C.c_int]
    L.sim_set_rank_stream_eager.argtypes = [C.c_int, C.c_int]
    L.fakecuda_set_all_eager(0)
    world, per, steps = 2, 4, 3
    params, data, label = case(world * per, seed=13)
    L.sim_use_rank_stream(-1)
    L.sim_set_solver_count(1)
    one = trainer(sim_host, world * per, params, data, label)
    one_losses = []
    for _ in range(steps):
        one.step(1)
        one_losses.append(one.loss())
    one_p = [one.get_param(i, 0) for i in range(6)]
    try:
        ranks, uid = [], None
        for r in range(world):
            L.sim_use_rank_stream(r)
            t = trainer(sim_host, per, [p if r == 0 else p + np.float32(0.5) for p in params],
                        data[r * per:(r + 1) * per], label[r * per:(r + 1) * per])
            if r == 0:
                uid = t.new_unique_id()
            t.attach_sync(world, r, uid)
            ranks.append(t)
        compute_eager, side_eager = STEP_MODES[mode]
        L.fakecuda_set_all_eager(side_eager)
        for r in range(world):
            L.sim_set_rank_stream_eager(r, compute_eager)
        losses = [[] for _ in range(world)]
        for _ in range(steps):
            for r, t in enumerate(ranks):
                L.sim_use_rank_stream(r)
                t.step(1)
            for r, t in enumerate(ranks):
                L.sim_use_rank_stream(r)
                losses[r].append(t.loss())
        out = []
        for r, t in enumerate(ranks):
            L.sim_use_rank_stream(r)
            out.append(([t.get_param(i, 0) for i in range(6)], [t.get_param(i, 2) for i in range(6)]))
    finally:
        L.sim_use_rank_stream(-1)
        L.fakecuda_set_all_eager(0)
        L.sim_set_solver_count(1)
    for i in range(6):
        assert np.array_equal(out[0][0][i].view(np.uint32), out[1][0][i].view(np.uint32)), i
        assert np.array_equal(out[0][1][i].view(np.uint32), out[1][1][i].view(np.uint32)), i
        assert rel(out[0][0][i], one_p[i]) < 1e-5, i
    np.testing.assert_allclose(np.mean(losses, axis=0), one_losses, rtol=1e-5)

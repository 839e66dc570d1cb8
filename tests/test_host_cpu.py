"""CPU tests of the C++ host layer (libb2caffe.so): registry, solver schedules, bucket plan, batch division.
These mirror test_layer_factory.cpp / the schedule part of test_gradient_based_solver.cpp; no GPU needed."""
import numpy as np
import pytest

import oracle as o
from caffe_mpi_b200 import host_api as h


def test_layer_registry_knows_convolution():
    assert h.lib().b2h_registry_has(b"Convolution") == 1
    assert h.lib().b2h_registry_has(b"NoSuchLayer") == 0


POLICIES = [
    dict(lr_policy="fixed", base_lr=0.01),
    dict(lr_policy="step", base_lr=0.1, gamma=0.5, stepsize=10),
    dict(lr_policy="exp", base_lr=0.1, gamma=0.999),
    dict(lr_policy="inv", base_lr=0.01, gamma=1e-4, power=0.75),                     # examples/mnist/lenet_solver
    dict(lr_policy="poly", base_lr=0.001, power=2.0, max_iter=2400000),              # models/resnet50/solver.prototxt
    dict(lr_policy="sigmoid", base_lr=0.1, gamma=-0.01, stepsize=50),
    dict(lr_policy="fixed", base_lr=0.1, rampup_interval=20, rampup_lr=0.01),
]


@pytest.mark.parametrize("cfg", POLICIES, ids=[c["lr_policy"] + str(i) for i, c in enumerate(POLICIES)])
def test_learning_rate_matches_oracle(cfg):
    s = h.SGDSolver(**cfg)
    for it in (0, 1, 5, 19, 20, 37, 100, 1234):
        want = o.learning_rate(cfg["lr_policy"], it, cfg["base_lr"], cfg.get("gamma", 0.1), cfg.get("power", 1.0),
                               cfg.get("stepsize", 1), cfg.get("max_iter", 1), cfg.get("min_lr", 0.0), 0,
                               cfg.get("rampup_interval", 0), cfg.get("rampup_lr", 0.0))
        assert s.lr_at(it) == pytest.approx(want, rel=1e-6, abs=1e-12)


def test_multistep_policy():
    s = h.SGDSolver(lr_policy="multistep", base_lr=0.1, gamma=0.1, stepvalue=[10, 20])
    got = [s.lr_at(i) for i in (0, 9, 10, 15, 20, 25)]          # iterations visited in order, like Solver::Step
    assert got == pytest.approx([0.1, 0.1, 0.01, 0.01, 0.001, 0.001], rel=1e-5)


def test_unknown_policy_is_fatal():
    s = h.SGDSolver(lr_policy="bogus")
    with pytest.raises(h.HostError, match="Unknown learning rate policy"):
        s.lr_at(0)


def reference_bucket_walk(counts, reduce_buckets):
    """Independent restatement of Net::ReduceAndUpdate's bucketing (net.cpp:772-783,824-862) for ids arriving
    last-to-first."""
    even = lambda c: c + (c & 1)
    n = len(counts)
    space = sum(even(c) for c in counts)
    mppb = max(1, (n + 1) // reduce_buckets)
    bsc = int(np.float32(space + 1) / np.float32(n) * np.float32(mppb))
    out, lo, hi, rec = [], -1, -1, 0
    for pid in range(n - 1, -1, -1):
        if rec >= bsc or (lo != -1 and pid < lo - 1) or (hi != -1 and pid > hi + 1):
            out.append((lo, hi))
            lo = hi = pid
            rec = even(counts[pid])
        else:
            lo = pid if lo == -1 or pid < lo else lo
            hi = pid if hi == -1 or pid > hi else hi
            rec += even(counts[pid])
    if lo != -1:
        out.append((lo, hi))
    return out


@pytest.mark.parametrize("seed", range(5))
def test_bucket_plan_matches_reference_walk(seed):
    rng = np.random.default_rng(seed)
    counts = [int(c) for c in rng.integers(1, 300000, size=int(rng.integers(1, 170)))]
    for rb in (1, 2, 6, 50):
        plan = h.plan_buckets(counts, rb)
        assert [(f, t) for f, t, _, _ in plan] == reference_bucket_walk(counts, rb)
        # buckets tile the arena exactly: contiguous, even-padded, every param in exactly one bucket
        even = lambda c: c + (c & 1)
        offs = np.cumsum([0] + [even(c) for c in counts])
        seen = []
        for f, t, off, cnt in plan:
            assert off == offs[f] and cnt == offs[t + 1] - offs[f]
            seen += list(range(f, t + 1))
        assert sorted(seen) == list(range(len(counts)))


def test_resnet50_bucket_sizes():
    # 161 reduced blobs, 102.2 MB arena, reduce_buckets = 6 -> messages of roughly 1/6 of the arena (SURVEY 2.3)
    from caffe_mpi_b200.shapes import RESNET50
    counts = []
    for (cnt, C, H, O, k, s, p, G, b) in RESNET50:
        for _ in range(cnt):
            counts += [O * (C // G) * k * k, O, O]       # conv W + BN scale + BN bias
    counts += [2048 * 1000, 1000]
    plan = h.plan_buckets(counts, 6)
    assert 4 <= len(plan) <= 12
    assert sum(c for *_, c in plan) == sum(c + (c & 1) for c in counts)


def test_divide_batch_size():
    # parallel.cpp:284-293: per-rank batch = total / solver_count rounded up
    assert h.divide_batch_size(512, 8) == 64
    assert h.divide_batch_size(100, 8) == 13
    assert h.divide_batch_size(32, 1) == 32


MOMENTA = [
    dict(momentum_policy="fixed", momentum=0.9),
    dict(momentum_policy="fixed", momentum=0.9, max_momentum=0.5),                      # "fixed" ignores max_momentum
    dict(momentum_policy="poly", momentum=0.5, max_momentum=0.95, momentum_power=2.0),
    dict(momentum_policy="poly", momentum=0.5),                                           # max_momentum's default, 0.99
    dict(momentum_policy="poly", momentum=0.9, max_momentum=0.999, momentum_power=0.5),
    dict(momentum_policy="opt", momentum=0.9),                                            # no clamp
    dict(momentum_policy="opt", momentum=0.9, max_momentum=0.99),
    dict(momentum_policy="opt", momentum=0.9, max_momentum=0.995),
]


@pytest.mark.parametrize("cfg", MOMENTA, ids=[f'{c["momentum_policy"]}{i}' for i, c in enumerate(MOMENTA)])
@pytest.mark.parametrize("lr", [0.01, 2e-4, 1e-4, 5e-5, 1e-6])
def test_momentum_policy_matches_oracle(cfg, lr):
    """SGDSolver::GetMomentum against the oracle's restatement of the reference (sgd_solver.cpp:68-91), at learning rates on both
    sides of 1.0e-4, where the "opt" momentum (1 - sqrt(lr)/2)^2 crosses 0.99; max_momentum clamps "opt" only when it is given"""
    fields = " ".join(f'{k}: "{v}"' if isinstance(v, str) else f"{k}: {v!r}" for k, v in cfg.items())
    s, _ = h.open_solver(f'type: "SGD" base_lr: {lr!r} lr_policy: "fixed" max_iter: 100 {fields}', is_text=True)
    for it in (0, 1, 10, 50, 99, 100):
        want = o.momentum(cfg["momentum_policy"], it, cfg["momentum"], cfg.get("max_momentum", 0.99), "max_momentum" in cfg,
                          cfg.get("momentum_power", 1.0), 100, s.lr_at(it))
        if cfg["momentum_policy"] == "poly":
            assert s.momentum_at(it) == pytest.approx(want, rel=1e-6), it
        else:
            assert s.momentum_at(it) == want, it
    if cfg["momentum_policy"] == "opt":
        free = float(np.float32((1.0 - 0.5 * float(np.sqrt(np.float32(lr)))) ** 2))
        clamp = cfg.get("max_momentum", np.inf)
        assert s.momentum_at(0) == pytest.approx(min(free, clamp), rel=1e-7)
        if "max_momentum" not in cfg and lr <= 5e-5:
            assert s.momentum_at(0) > 0.99                 # the reference does not clamp without max_momentum


def test_opt_momentum_follows_the_learning_rate_schedule():
    """"opt" reads GetLearningRate at the same iteration: a step schedule takes lr from 1e-2 through 1e-4 to 1e-6"""
    s, _ = h.open_solver('type: "SGD" base_lr: 0.01 lr_policy: "step" gamma: 0.01 stepsize: 10 max_iter: 30 momentum: 0.9 '
                         'momentum_policy: "opt"', is_text=True)
    got = [s.momentum_at(it) for it in (0, 10, 20)]
    want = [o.momentum("opt", it, 0.9, lr=s.lr_at(it)) for it in (0, 10, 20)]
    assert got == want
    assert got[0] == pytest.approx(0.95 ** 2, rel=1e-6) and got[2] == pytest.approx(0.9995 ** 2, rel=1e-6)


def test_unknown_momentum_policy_is_fatal():
    s, _ = h.open_solver('type: "SGD" base_lr: 0.01 momentum: 0.9 momentum_policy: "bogus"', is_text=True)
    with pytest.raises(h.HostError, match="Unknown momentum policy"):
        s.momentum_at(0)

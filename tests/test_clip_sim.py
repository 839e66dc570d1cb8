"""clip_gradients through the whole C++ host layer without a GPU: TrainNet, the bucketed ReduceScheduler with the norm's partials on the
side stream, the factor and the one whole-arena update behind the last bucket, P2PSync -- on the stream-order model of the CUDA runtime
(tests/sim/fake_cuda.cpp) with the host stand-ins of tests/sim/fake_kernels_clip.cpp (libclipsim.so, tests/sim/Makefile.clip).
References: tests/netoracle.py forward / backward, the clip oracle tests/clip_oracle.py and the solver oracle tests/solver_oracle.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from caffe_mpi_b200 import capi
import clip_oracle as co
import netoracle as no
from test_solvers_gpu import _hp, make_trainer, rel, solver_text
from test_trainer_sim import STEP_MODES, _set_modes

HERE = os.path.dirname(os.path.abspath(__file__))
BASE_LR = {"SGD": 0.05, "Adam": 0.001}


@pytest.fixture(scope="module")
def clip_sim():
    """host_api pointed at libclipsim.so for the duration of the module."""
    from caffe_mpi_b200 import host_api
    capi.lib()
    r = subprocess.run(["make", "-C", os.path.join(HERE, "sim"), "-f", "Makefile.clip", "libclipsim.so"], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.fail("tests/sim/libclipsim.so does not build:\n" + r.stdout[-1000:] + r.stderr[-3000:])
    saved = (host_api._lib, host_api._SO, os.environ.get("B2C_NCCL_ARENA"))
    host_api._lib, host_api._SO = None, os.path.join(HERE, "sim", "libclipsim.so")
    os.environ["B2C_NCCL_ARENA"] = "0"
    L = host_api.lib()
    for fn, at in (("sim_use_rank_stream", [C.c_int]), ("fakecuda_set_all_eager", [C.c_int]), ("sim_set_solver_count", [C.c_int]),
                   ("fakecuda_set_eager", [C.c_void_p, C.c_int]), ("sim_set_rank_stream_eager", [C.c_int, C.c_int])):
        getattr(L, fn).argtypes = at
    try:
        yield host_api
    finally:
        L.sim_use_rank_stream(-1)
        L.fakecuda_set_all_eager(0)
        L.sim_set_solver_count(1)
        host_api._lib, host_api._SO = saved[0], saved[1]
        if saved[2] is None:
            os.environ.pop("B2C_NCCL_ARENA", None)
        else:
            os.environ["B2C_NCCL_ARENA"] = saved[2]


def _spec(net):
    return no.mini_resnet() if net == "resnet" else no.lenet(batch=8)


def _clip_between(kind, spec, steps=3):
    """a clip between the unclipped run's smallest and largest norm, so that some steps clip and some do not"""
    params, data, label = _case(spec)
    norms = co.replay(kind, spec, params, data, label, steps, BASE_LR[kind], 1e30, _hp(kind))[4]
    return float(np.median(norms)) * 1.001, norms            # the median step's norm stays clear of the clip


def _case(spec):
    rng = np.random.default_rng(1701)
    params = []
    for _, pk, shp in no.param_shapes(spec):
        params.append((rng.standard_normal(shp) * np.sqrt(2.0 / np.prod(shp[1:]))).astype(np.float32) if pk == "w" else
                      rng.uniform(0.5, 1.5, shp).astype(np.float32) if pk == "scale" else rng.uniform(-0.2, 0.2, shp).astype(np.float32))
    data = rng.standard_normal(spec[0]["shape"]).astype(np.float32)
    label = rng.integers(0, 10, spec[0]["shape"][0]).astype(np.float32)
    return params, data, label


def _trainer(host, spec, solver, net_prefix=""):
    params, data, label = _case(spec)
    t = host.Trainer(net_prefix + no.to_prototxt(spec), solver, num_classes=10)
    for i, p in enumerate(params):
        t.set_param(i, p)
    t.set_blob("data", data)
    t.set_blob("label", label)
    return t, params, data, label


def _state(t, n, two=True):
    return [[t.get_param(i, k).copy() for i in range(n)] for k in ((0, 2, 3) if two else (0, 2))]


@pytest.mark.parametrize("mode", sorted(STEP_MODES))
@pytest.mark.parametrize("net", ["resnet", "lenet"])
@pytest.mark.parametrize("kind", ["SGD", "Adam"])
def test_clipped_steps_under_extreme_stream_orders(clip_sim, kind, net, mode):
    """Three clipped Solver::Step iterations under each extreme stream order against the replay: every loss, norm, parameter and
    history; the clip is such that some steps clip and some do not"""
    L = clip_sim.lib()
    L.fakecuda_set_all_eager(0)
    spec = _spec(net)
    clip, norms = _clip_between(kind, spec)
    clipped = sum(1 for n in norms if n > np.float32(clip))
    assert 0 < clipped < 3, norms
    t, params, data, label = _trainer(clip_sim, spec, solver_text(kind, BASE_LR[kind]) + " clip_gradients: %r" % clip)
    _set_modes(L, mode)
    try:
        ref_losses, ref_p, ref_h, ref_h2, ref_norms = co.replay(kind, spec, params, data, label, 3, BASE_LR[kind], clip, _hp(kind))
        losses, got_norms = [], []
        for _ in range(3):
            t.step(1)
            losses.append(t.loss())
            got_norms.append(t.clip_state()[0])
        np.testing.assert_allclose(losses, ref_losses, rtol=2e-4)
        np.testing.assert_allclose(got_norms, ref_norms, rtol=2e-4)
        assert all(abs(n - clip) > 1e-4 * clip for n in ref_norms)
        assert t.clip_state()[2] == sum(1 for n in ref_norms if n > np.float32(clip))
        hf = 1e-3 * max(float(np.abs(x).max()) for x in ref_h)
        for i in range(len(ref_p)):
            assert rel(t.get_param(i, 0), ref_p[i]) <= 2e-4, (kind, mode, i)
            assert rel(t.get_param(i, 2), ref_h[i], hf) <= 5e-4, (kind, mode, i)
            assert not t.get_param(i, 1).any()
    finally:
        L.fakecuda_set_all_eager(0)


@pytest.mark.parametrize("mode", ["all-lazy", "compute-lazy_side-eager"])
def test_bucket_plans_give_identical_bits(clip_sim, mode):
    """reduce_buckets 1, 6 and one bucket per parameter: the partials depend only on each segment, so every weight and history bit
    is the same"""
    L = clip_sim.lib()
    spec = no.mini_resnet()
    clip, _ = _clip_between("Adam", spec)
    solver = solver_text("Adam", BASE_LR["Adam"]) + " clip_gradients: %r" % clip
    out = []
    for rb in (1, 6, 1000):
        L.fakecuda_set_all_eager(0)
        t, params, _, _ = _trainer(clip_sim, spec, solver, "reduce_buckets: %d\n" % rb)
        _set_modes(L, mode)
        try:
            t.step(3)
            out.append((_state(t, len(params)), t.clip_state()))
        finally:
            L.fakecuda_set_all_eager(0)
    for o in out[1:]:
        assert o[1] == out[0][1]
        for k in range(3):
            for a, b in zip(out[0][0][k], o[0][k]):
                assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


def test_iter_size_clips_the_accumulated_sum(clip_sim):
    spec = no.lenet(batch=8)
    kind = "SGD"
    params, data, label = _case(spec)
    norms = co.replay(kind, spec, params, data, label, 3, BASE_LR[kind], 1e30, _hp(kind), iter_size=2)[4]
    clip = float(np.median(norms)) * 1.001
    t, params, data, label = _trainer(clip_sim, spec, solver_text(kind, BASE_LR[kind]) + " iter_size: 2 clip_gradients: %r" % clip)
    ref_losses, ref_p, _, _, ref_norms = co.replay(kind, spec, params, data, label, 3, BASE_LR[kind], clip, _hp(kind), iter_size=2)
    got = []
    for _ in range(3):
        t.step(1)
        got.append(t.clip_state()[0])
    np.testing.assert_allclose(got, ref_norms, rtol=2e-4)
    assert 0 < t.clip_state()[2] < 3
    for i in range(len(ref_p)):
        assert rel(t.get_param(i, 0), ref_p[i]) <= 2e-4, i


@pytest.mark.parametrize("kind", ["SGD", "Adam"])
def test_huge_clip_is_bitwise_no_clip(clip_sim, kind):
    L = clip_sim.lib()
    L.fakecuda_set_all_eager(0)
    spec = no.mini_resnet()
    out = []
    for extra in ("", " clip_gradients: 1e30"):
        t, params, _, _ = _trainer(clip_sim, spec, solver_text(kind, BASE_LR[kind]) + extra)
        t.step(3)
        out.append(_state(t, len(params), kind == "Adam"))
    for k in (0, 1):
        for a, b in zip(out[0][k], out[1][k]):
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("mode", sorted(STEP_MODES))
@pytest.mark.parametrize("world", [2, 3])
def test_n_solvers_equal_one_solver_on_the_full_batch(clip_sim, world, mode):
    """`world` TrainNets in one process through P2PSync: the norm is taken of the reduced gradient (s_n = 1/world), so every rank
    computes the same factor -- bit-identical ranks -- and they equal one solver on the whole batch"""
    import multi_rank_worker as mw
    L = clip_sim.lib()
    L.fakecuda_set_all_eager(0)
    kind = "Adam"
    global_batch, steps = 6 * world, 3
    params, data, label = mw.build_case(global_batch)
    solver = solver_text(kind, BASE_LR[kind]) + " clip_gradients: 0.5"

    def trainer(batch, ps, d, lb):
        t = clip_sim.Trainer(no.to_prototxt(no.lenet(batch=batch)), solver, num_classes=10)
        for i, p in enumerate(ps):
            t.set_param(i, p)
        t.set_blob("data", d)
        t.set_blob("label", lb)
        return t
    L.sim_use_rank_stream(-1)
    L.sim_set_solver_count(1)
    one = trainer(global_batch, params, data, label)
    one.step(steps)
    ref = _state(one, len(params))
    ref_clip = one.clip_state()
    assert ref_clip[2] > 0
    per = global_batch // world
    try:
        ranks, uid = [], None
        for r in range(world):
            L.sim_use_rank_stream(r)
            t = trainer(per, [p if r == 0 else p + np.float32(0.5 + r) for p in params], data[r * per:(r + 1) * per],
                        label[r * per:(r + 1) * per])
            if r == 0:
                uid = t.new_unique_id()
            t.attach_sync(world, r, uid)
            ranks.append(t)
        compute_eager, side_eager = STEP_MODES[mode]
        L.fakecuda_set_all_eager(side_eager)
        for r in range(world):
            L.sim_set_rank_stream_eager(r, compute_eager)
        for _ in range(steps):
            for r, t in enumerate(ranks):
                L.sim_use_rank_stream(r)
                t.step(1)
        out, clips = [], []
        for r, t in enumerate(ranks):
            L.sim_use_rank_stream(r)
            out.append(_state(t, len(params)))
            clips.append(t.clip_state())
    finally:
        L.sim_use_rank_stream(-1)
        L.fakecuda_set_all_eager(0)
        L.sim_set_solver_count(1)
    assert all(c == clips[0] for c in clips) and clips[0][2] == ref_clip[2]
    assert abs(clips[0][0] - ref_clip[0]) <= 1e-5 * ref_clip[0]
    for k, name in enumerate(("param", "history", "history2")):
        floor = 1e-3 * max(float(np.abs(x).max()) for x in ref[k])
        for i in range(len(params)):
            for r in range(1, world):
                assert np.array_equal(out[0][k][i].view(np.uint32), out[r][k][i].view(np.uint32)), f"{name} {i} differs on rank {r}"
            assert rel(out[0][k][i], ref[k][i], floor) < (1e-5 if k == 0 else 1e-4), (name, i)


def test_standalone_solver_clips_through_the_scheduler(clip_sim):
    """the standalone solver handle steps through the same ReduceScheduler: its buckets take norm partials, then one factor and one
    update of the whole arena"""
    s = clip_sim.SGDSolver(base_lr=0.1, momentum=0.9, clip_gradients=1.0, reduce_buckets=3)
    s.set_params([10, 6, 4])
    g = [np.full(10, 0.3, np.float32), np.full(6, 0.4, np.float32), np.full(4, -0.5, np.float32)]
    for i, x in enumerate(g):
        s.set(i, x, diff=True)
    s.step()
    norm, factor, n = s.clip_state()
    want_norm, want_factor = co.clip_factor(g, 1.0)
    assert (np.float32(norm), np.float32(factor), n) == (want_norm, want_factor, 1)
    for i, x in enumerate(g):
        np.testing.assert_array_equal(s.get(i, 0), -(np.float32(0.1) * (x * want_factor)))
    L = clip_sim.lib()
    assert L.b2h_solver_set_clip_gradients(s._h, 2.0) == -1 and b"before the solver's parameters" in L.b2h_last_error()

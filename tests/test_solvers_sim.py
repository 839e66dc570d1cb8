"""The Nesterov, AdaGrad, RMSProp, AdaDelta and Adam solvers through the whole C++ host layer without a GPU: TrainNet, the parameter arena
with its second history, the bucketed ReduceScheduler, P2PSync and Snapshot / Restore on the stream-order model of the CUDA runtime
(tests/sim/fake_cuda.cpp), with the update itself run by the host stand-in tests/sim/fake_kernels_solvers.cpp (libsolversim.so,
tests/sim/Makefile.solvers).  References: tests/netoracle.py forward / backward and the fp32 solver oracle tests/solver_oracle.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from caffe_mpi_b200 import capi, host_api
import caffe_state_proto as csp
import netoracle as no
import solver_oracle as so
from test_solvers_gpu import _hp, make_trainer, rel, solver_text
from test_trainer_sim import STEP_MODES, _set_modes

HERE = os.path.dirname(os.path.abspath(__file__))
NEW_KINDS = ("Nesterov", "AdaGrad", "RMSProp", "AdaDelta", "Adam")
# the normalising solvers step by about base_lr for any gradient well above delta; small rates keep a ReLU unit that flips between
# the two computations from dominating the comparison (tests/test_solvers_gpu.py::test_steps_match_net_oracle)
BASE_LR = {"Nesterov": 0.05, "AdaGrad": 0.001, "RMSProp": 0.001, "AdaDelta": 0.05, "Adam": 0.001}


@pytest.fixture(scope="module")
def solver_sim():
    """host_api pointed at libsolversim.so for the duration of the module."""
    capi.lib()
    r = subprocess.run(["make", "-C", os.path.join(HERE, "sim"), "-f", "Makefile.solvers", "libsolversim.so"], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.fail("tests/sim/libsolversim.so does not build:\n" + r.stdout[-1000:] + r.stderr[-3000:])
    saved = (host_api._lib, host_api._SO, os.environ.get("B2C_NCCL_ARENA"))
    host_api._lib, host_api._SO = None, os.path.join(HERE, "sim", "libsolversim.so")
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


def replay(kind, spec, params, data, label, steps, base_lr):
    """netoracle forward / backward + the solver oracle, lr_policy fixed, weight_decay 0.0005: (losses, params, h, h2)."""
    hp = _hp(kind)
    p = [x.copy() for x in params]
    h = [np.zeros(x.size, np.float32) for x in params]
    h2 = [np.zeros(x.size, np.float32) for x in params]
    losses = []
    for it in range(steps):
        loss, grads, _, _ = no.forward_backward(spec, p, data, label)
        losses.append(loss)
        for i, g in enumerate(grads):
            _, w, h[i], b = so.update(kind, g, p[i], h[i], h2[i], hp, base_lr, 0.0005, t=it + 1)
            p[i] = w.reshape(p[i].shape)
            if b is not None:
                h2[i] = b
    return losses, p, h, h2


@pytest.mark.parametrize("mode", sorted(STEP_MODES))
@pytest.mark.parametrize("net", ["resnet", "lenet"])
@pytest.mark.parametrize("kind", NEW_KINDS)
def test_steps_under_extreme_stream_orders(solver_sim, kind, net, mode):
    """Three Solver::Step iterations (forward, backward, per-bucket update on the side stream, the event hand-overs) under each extreme
    stream order against the replay: losses, parameters, both histories, cleared diffs."""
    L = solver_sim.lib()
    L.fakecuda_set_all_eager(0)
    spec = no.mini_resnet() if net == "resnet" else no.lenet(batch=8)
    t, params, data, label = make_trainer(spec, solver_text(kind, BASE_LR[kind]), np.random.default_rng(1701))
    _set_modes(L, mode)
    try:
        ref_losses, ref_p, ref_h, ref_h2 = replay(kind, spec, params, data, label, 3, BASE_LR[kind])
        losses = []
        for k in range(3):
            t.step(1)
            if k != 1:                                     # the second step starts with the first one's loss never read
                losses.append(t.loss())
        np.testing.assert_allclose(losses, [ref_losses[0], ref_losses[2]], rtol=2e-4)
        two = kind in so.TWO_HISTORIES
        hf = 1e-3 * max(float(np.abs(x).max()) for x in ref_h)
        h2f = 1e-3 * max(float(np.abs(x).max()) for x in ref_h2) if two else 0
        for i in range(len(ref_p)):
            assert rel(t.get_param(i, 0), ref_p[i]) <= 2e-4, (kind, mode, i)
            assert rel(t.get_param(i, 2), ref_h[i], hf) <= 5e-4, (kind, mode, i)
            if two:
                assert rel(t.get_param(i, 3), ref_h2[i], h2f) <= 5e-4, (kind, mode, i)
            assert not t.get_param(i, 1).any()
    finally:
        L.fakecuda_set_all_eager(0)


def _lenet_trainer(host, kind, batch, params, data, label):
    t = host.Trainer(no.to_prototxt(no.lenet(batch=batch)), solver_text(kind, BASE_LR[kind]), num_classes=10)
    for i, p in enumerate(params):
        t.set_param(i, p)
    t.set_blob("data", data)
    t.set_blob("label", label)
    return t


@pytest.mark.parametrize("mode", sorted(STEP_MODES))
@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("kind", ["Adam", "AdaDelta"])
def test_n_solvers_equal_one_solver_on_the_full_batch(solver_sim, kind, world, mode):
    """`world` TrainNets in one process, each with its own streams and P2PSync, train LeNet on their slices of one global batch through
    the bucketed allreduce (a collective of the stream-order model) and the fused update: every rank ends with the same parameters and
    both histories bit for bit, and those equal one solver on the whole batch."""
    import multi_rank_worker as mw
    L = solver_sim.lib()
    L.fakecuda_set_all_eager(0)
    global_batch, steps = 6 * world, 3
    params, data, label = mw.build_case(global_batch)
    per = global_batch // world
    L.sim_use_rank_stream(-1)
    L.sim_set_solver_count(1)
    one = _lenet_trainer(solver_sim, kind, global_batch, params, data, label)
    for _ in range(steps):
        one.step(1)
    ref = [[one.get_param(i, k) for i in range(len(params))] for k in (0, 2, 3)]
    try:
        ranks = []
        uid = None
        for r in range(world):
            L.sim_use_rank_stream(r)
            t = _lenet_trainer(solver_sim, kind, per, [p if r == 0 else p + np.float32(0.5 + r) for p in params],
                               data[r * per:(r + 1) * per], label[r * per:(r + 1) * per])
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
        out = []
        for r, t in enumerate(ranks):
            L.sim_use_rank_stream(r)
            out.append([[t.get_param(i, k) for i in range(len(params))] for k in (0, 2, 3)])
    finally:
        L.sim_use_rank_stream(-1)
        L.fakecuda_set_all_eager(0)
        L.sim_set_solver_count(1)
    for k, name in enumerate(("param", "history", "history2")):
        floor = 1e-3 * max(float(np.abs(x).max()) for x in ref[k])
        for i in range(len(params)):
            for r in range(1, world):
                assert np.array_equal(out[0][k][i].view(np.uint32), out[r][k][i].view(np.uint32)), f"{name} {i} differs on rank {r}"
            assert rel(out[0][k][i], ref[k][i], floor) < (1e-5 if k == 0 else 1e-4), (name, i)


@pytest.mark.parametrize("kind", ["Adam", "AdaDelta"])
def test_snapshot_restore_step_is_bitwise_and_the_state_has_the_reference_layout(solver_sim, kind, tmp_path):
    """step, snapshot, step  ==  fresh trainer, restore, step, bit for bit.  The .solverstate, read with google.protobuf against the
    reference's message definitions, holds 2 * np history blobs in AdamPreSolve's order [h_0 .. h_np-1, h2_0 .. h2_np-1]; and a state
    the reference's way of writing (packed `data`, no raw bytes) restores into both histories."""
    import multi_rank_worker as mw
    L = solver_sim.lib()
    L.fakecuda_set_all_eager(0)
    params, data, label = mw.build_case(8)
    t = _lenet_trainer(solver_sim, kind, 8, params, data, label)
    t.step(2)
    h_at2 = [[t.get_param(i, k).copy() for i in range(len(params))] for k in (2, 3)]
    state = t.snapshot(str(tmp_path / "snap"))
    t.step(2)
    want = [[t.get_param(i, k).copy() for i in range(len(params))] for k in (0, 2, 3)]
    it, _, learned, blobs = csp.read_state(state)
    n = t.num_learnable()
    assert it == 2 and learned.endswith("_iter_2.caffemodel") and n == len(params) and len(blobs) == 2 * n
    for i in range(n):                                    # LeNet: every learnable blob is trainable, in the same order
        assert np.array_equal(blobs[i].view(np.uint32), h_at2[0][i].view(np.uint32)), ("h", i)
        assert np.array_equal(blobs[n + i].view(np.uint32), h_at2[1][i].view(np.uint32)), ("h2", i)
    t2 = _lenet_trainer(solver_sim, kind, 8, [p + np.float32(1) for p in params], data, label)
    t2.restore(state)
    assert t2.iter() == 2
    t2.step(2)
    for k, what in enumerate((0, 2, 3)):
        for i in range(n):
            assert np.array_equal(t2.get_param(i, what).view(np.uint32), want[k][i].view(np.uint32)), (what, i)
    # a reference-layout state written by an independent encoder
    rng = np.random.default_rng(3)
    hs = [rng.standard_normal(p.size).astype(np.float32) for p in params] + [np.abs(rng.standard_normal(p.size)).astype(np.float32) for p in params]
    ref_state = str(tmp_path / "ref.solverstate")
    csp.write_state(ref_state, 7, "", hs, [p.shape for p in params] * 2)
    t3 = _lenet_trainer(solver_sim, kind, 8, params, data, label)
    t3.restore(ref_state)
    assert t3.iter() == 7
    for i in range(n):
        assert np.array_equal(t3.get_param(i, 2).view(np.uint32), hs[i].view(np.uint32))
        assert np.array_equal(t3.get_param(i, 3).view(np.uint32), hs[n + i].view(np.uint32))
    # and the one-history layout does not restore into a two-history solver
    csp.write_state(str(tmp_path / "short.solverstate"), 7, "", hs[:n], [p.shape for p in params])
    with pytest.raises(host_api.HostError, match="Incorrect length of history blobs"):
        t3.restore(str(tmp_path / "short.solverstate"))

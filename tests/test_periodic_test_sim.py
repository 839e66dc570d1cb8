"""Periodic testing without a GPU: LeNet trained by 1, 2 and 3 in-process ranks (TrainNet + P2PSync over tests/sim/fake_comm.cpp, one
compute stream each) with a weight-sharing TEST net on a TEST LMDB, scored by TrainNet's test pass (device score vector, one score
allreduce on the comm stream, one read) under the four extreme stream orders of tests/sim/fake_cuda.cpp.  Every rank must get the
same means, equal to the numpy TEST forward (tests/infer_oracle.py) on the current weights over the union of the ranks' stripes,
and the passes must leave every weight and history bit of training untouched."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from caffe_mpi_b200 import capi, host_api
import infer_oracle as io_
import netoracle as no
from test_data_cpu import oracle_batches

HERE = os.path.dirname(os.path.abspath(__file__))
SOLVER = 'base_lr: 0.05 lr_policy: "fixed" momentum: 0.9 weight_decay: 0.0005 max_iter: 100 solver_mode: GPU'
STEP_MODES = {"all-lazy": (0, 0), "all-eager": (1, 1), "compute-lazy_side-eager": (0, 1), "compute-eager_side-lazy": (1, 0)}
SCALE = 0.00390625


@pytest.fixture(scope="module")
def sim_host():
    """host_api pointed at libtestpasssim.so (libtrainsim.so plus the two halves of the test pass) for the duration of the module."""
    capi.lib()
    r = subprocess.run(["make", "-C", os.path.join(HERE, "sim"), "-f", "Makefile.testpass", "libtestpasssim.so"], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.fail("tests/sim/libtestpasssim.so does not build:\n" + r.stdout[-1000:] + r.stderr[-3000:])
    saved = (host_api._lib, host_api._SO, os.environ.get("B2C_NCCL_ARENA"))
    host_api._lib, host_api._SO = None, os.path.join(HERE, "sim", "libtestpasssim.so")
    os.environ["B2C_NCCL_ARENA"] = "0"
    try:
        L = host_api.lib()
        for fn, at in (("sim_use_rank_stream", [C.c_int]), ("fakecuda_set_all_eager", [C.c_int]), ("sim_set_solver_count", [C.c_int]),
                       ("sim_set_rank_stream_eager", [C.c_int, C.c_int]), ("sim_tester_enqueue_pass", [C.c_void_p, C.c_int]),
                       ("sim_tester_read_pass", [C.c_void_p, C.c_void_p, C.POINTER(C.c_float)])):
            getattr(L, fn).argtypes = at
        L.sim_pass_last_error.restype = C.c_char_p
        yield host_api
    finally:
        host_api._lib, host_api._SO = saved[0], saved[1]
        if saved[2] is None:
            os.environ.pop("B2C_NCCL_ARENA", None)
        else:
            os.environ["B2C_NCCL_ARENA"] = saved[2]


def lenet_with_databases(train, test, batch, test_batch):
    """LeNet (no.lenet) fed by a TRAIN and a TEST Data layer, with the TEST-phase Accuracy layer of lenet_train_test.prototxt."""
    body = [ln for ln in no.to_prototxt(no.lenet()).splitlines() if 'type: "Input"' not in ln and not ln.startswith("name:")]
    data = ''.join(f'layer {{ name: "mnist" type: "Data" top: "data" top: "label" include {{ phase: {ph} }} transform_param {{ scale: {SCALE} }}\n'
                   f'  data_param {{ source: "{src}" batch_size: {b} backend: LMDB }} }}\n'
                   for ph, src, b in (("TRAIN", train, batch), ("TEST", test, test_batch)))
    acc = 'layer { name: "accuracy" type: "Accuracy" bottom: "ip2" bottom: "label" top: "accuracy" include { phase: TEST } }\n'
    return 'name: "LeNet"\n' + data + "\n".join(body) + "\n" + acc


@pytest.fixture(scope="module")
def databases(tmp_path_factory):
    from caffe_mpi_b200 import lmdb_io
    rng = np.random.default_rng(11)
    d = tmp_path_factory.mktemp("dbs")
    out = {}
    for name, n in (("train", 60), ("test", 48)):
        imgs = rng.integers(0, 256, (n, 1, 28, 28), dtype=np.uint8)
        labels = rng.integers(0, 10, n)
        lmdb_io.write_datum_lmdb(str(d / name), imgs, labels)
        out[name] = (str(d / name), imgs, labels)
    return out


B, TB, TEST_ITER, EVERY, STEPS = 2, 2, 2, 2, 4


def run_ranks(host, world, mode, net, with_tests):
    """Train `world` ranks for STEPS iterations in lockstep; with_tests: the shell's plan for test_interval EVERY (one batch at iteration
    0, TEST_ITER batches at every later multiple and after the last iteration), every rank's pass enqueued before any is read.
    Returns ([per pass: [per rank: (means, loss)]], [per pass: rank 0's trainable parameters when it ran], per rank: (params, history))."""
    L = host.lib()
    L.fakecuda_set_all_eager(0)
    L.sim_use_rank_stream(-1)
    L.sim_set_solver_count(1)
    passes, weights = [], []
    try:
        ranks, testers, uid = [], [], None
        for r in range(world):
            L.sim_use_rank_stream(r)
            t = host.Trainer(net, SOLVER, num_classes=10, seed=50 + r)
            if world > 1:
                if r == 0:
                    uid = t.new_unique_id()
                t.attach_sync(world, r, uid)
            ranks.append(t)
            if with_tests:
                te = host.Tester(net, num_classes=10, seed=50 + r)
                te.share_trained_layers_with(t)
                testers.append(te)
        compute_eager, side_eager = STEP_MODES[mode]
        L.fakecuda_set_all_eager(side_eager)
        for r in range(world):
            L.sim_set_rank_stream_eager(r, compute_eager)
        width = len(testers[0].outputs()) if testers else 0

        def test_pass(batches):
            for r, te in enumerate(testers):
                L.sim_use_rank_stream(r)
                assert L.sim_tester_enqueue_pass(te._h, batches) == batches, L.sim_pass_last_error().decode()
            got = []
            for r, te in enumerate(testers):
                L.sim_use_rank_stream(r)
                m, loss = np.empty(width, np.float32), C.c_float()
                assert L.sim_tester_read_pass(te._h, m.ctypes.data_as(C.c_void_p), C.byref(loss)) == 0, L.sim_pass_last_error().decode()
                got.append((m, loss.value))
            passes.append(got)
            L.sim_use_rank_stream(0)
            weights.append([ranks[0].get_param(i) for i in range(ranks[0].num_params())])

        for it in range(STEPS):
            if with_tests and (it == 0 or it % EVERY == 0):
                test_pass(1 if it == 0 else TEST_ITER)
            for r, t in enumerate(ranks):
                L.sim_use_rank_stream(r)
                t.step(1, copy_input=True)
        if with_tests and STEPS % EVERY == 0:
            test_pass(TEST_ITER)
        final = []
        for r, t in enumerate(ranks):
            L.sim_use_rank_stream(r)
            final.append(([t.get_param(i) for i in range(t.num_params())], [t.get_param(i, 2) for i in range(t.num_params())]))
    finally:
        L.sim_use_rank_stream(-1)
        L.fakecuda_set_all_eager(0)
        L.sim_set_solver_count(1)
    return passes, weights, final


@pytest.mark.parametrize("mode", sorted(STEP_MODES))
@pytest.mark.parametrize("world", [1, 2, 3])
def test_test_passes_score_the_union_of_the_stripes_and_leave_training_alone(sim_host, databases, monkeypatch, world, mode):
    from oracle import layers_oracle as lo
    monkeypatch.delenv("B2C_DATA", raising=False)
    (train, _, _), (test, timgs, tlabels) = databases["train"], databases["test"]
    net = lenet_with_databases(train, test, B, TB)
    passes, weights, final = run_ranks(sim_host, world, mode, net, True)
    _, _, plain = run_ranks(sim_host, world, mode, net, False)
    # (b) the passes change no weight or history bit, and every rank holds the same bits
    for r in range(world):
        for a, b in zip(final[r][0] + final[r][1], plain[0][0] + plain[0][1]):
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), (world, mode, r)
    # (a) identical means on every rank, equal to the numpy TEST forward over the records the ranks read together
    spec = no.lenet()
    shapes = [shp for _, _, shp in no.param_shapes(spec)]
    weights = [[p.reshape(s) for p, s in zip(ps, shapes)] for ps in weights]
    stripes = [oracle_batches(len(tlabels), 1 + 2 * TEST_ITER, TB, world, r, 1) for r in range(world)]
    first = 0
    assert len(passes) == 3
    for k, (got, params) in enumerate(zip(passes, weights)):
        batches = 1 if k == 0 else TEST_ITER
        pos = [p for g in range(first, first + batches) for r in range(world) for p, _ in stripes[r][g]]
        first += batches
        x = timgs[pos].astype(np.float32) * np.float32(SCALE)
        y = tlabels[pos].astype(np.float32)
        union = no.lenet(batch=len(pos))
        no.param_shapes(union)                                               # (sets the conv layers' shapes for this batch)
        v = io_.forward_test_phase(union, params, {}, x, y)
        want = [float(lo.accuracy(v["ip2"], y)), float(v["loss"])]            # outputs in name order: accuracy, loss
        for r in range(world):
            assert np.array_equal(got[r][0].view(np.uint32), got[0][0].view(np.uint32)) and got[r][1] == got[0][1], (k, r)
        assert abs(got[0][0][0] - want[0]) <= 1e-6, (k, got[0][0], want)
        assert abs(got[0][0][1] - want[1]) <= 1e-5 * abs(want[1]), (k, got[0][0], want)
        assert abs(got[0][1] - want[1]) <= 1e-5 * abs(want[1]), k             # loss = 1 * the loss output's mean


def test_one_rank_test_pass_is_test_bit_for_bit_and_stops_between_batches(sim_host, databases, monkeypatch):
    """On one GPU the device score vector adds in Test()'s order: the same means, bit for bit.  A `between` hook that answers False
    stops the pass before that batch (no result, no further batch read)."""
    monkeypatch.delenv("B2C_DATA", raising=False)
    L = sim_host.lib()
    L.sim_use_rank_stream(-1)
    L.sim_set_solver_count(1)
    L.fakecuda_set_all_eager(0)
    (train, _, _), (test, _, _) = databases["train"], databases["test"]
    net = lenet_with_databases(train, test, B, TB)
    t = sim_host.Trainer(net, SOLVER, num_classes=10)
    t.step(2, copy_input=True)
    a, b = sim_host.Tester(net, num_classes=10), sim_host.Tester(net, num_classes=10)
    a.share_trained_layers_with(t)
    b.share_trained_layers_with(t)
    _, means, _ = a.test(3)
    got, loss = b.test_pass(3)
    assert np.array_equal(got.view(np.uint32), means.view(np.uint32))
    assert loss == got[1]
    seen = []
    assert b.test_pass(3, between=lambda i: seen.append(i) or i < 1) is None
    assert seen == [0, 1] and b.database_batches() == 4

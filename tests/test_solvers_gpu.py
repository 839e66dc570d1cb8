"""The Nesterov, AdaGrad, RMSProp, AdaDelta and Adam updates on the GPU: b2c_solver_update_arena against the fp32 oracle
(tests/solver_oracle.py), typed solver handles over several iterations, whole-net training through TrainNet against the net oracle,
snapshot / restore with two history arenas, and `caffe.py train` on the reference's solver files."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import netoracle as no
import oracle
import solver_oracle as so
from caffe_mpi_b200 import capi, host_api

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "tests", "golden", "reference_models")
HP = dict(momentum=0.9, delta=1e-3, rms_decay=0.95, momentum2=0.999)
NEW_KINDS = ("Nesterov", "AdaGrad", "RMSProp", "AdaDelta", "Adam")


def _hp(kind):
    return dict(HP, momentum=0.0 if kind in ("AdaGrad", "RMSProp") else HP["momentum"])


def _layout(rng):
    """130 segments (two launches of at most 96): odd counts and odd offsets, so segment starts are 4-byte but not 16-byte aligned
    and both scalar peels and the float4 body run; one segment spans several blocks; gaps between segments must stay untouched."""
    counts = [int(c) for c in rng.integers(1, 300, 128)] + [40000, 7]
    offsets, off = [], 3
    for c in counts:
        offsets.append(off)
        off += c + int(rng.integers(0, 3))
    return offsets, counts, off


@pytest.mark.parametrize("kind", NEW_KINDS + ("SGD",))
@pytest.mark.parametrize("l2", [True, False], ids=["L2", "L1"])
@pytest.mark.parametrize("clear", [True, False], ids=["clear", "keep"])
@pytest.mark.parametrize("h2_shift", [0, 1], ids=["h2_aligned", "h2_shifted"])
def test_arena_update_matches_oracle(kind, l2, clear, h2_shift):
    import torch
    if h2_shift and kind not in so.TWO_HISTORIES:
        pytest.skip("one-history solver")
    rng = np.random.default_rng(1701)
    offsets, counts, total = _layout(rng)
    g = rng.standard_normal(total).astype(np.float32)
    w = rng.standard_normal(total).astype(np.float32)
    h = np.abs(rng.standard_normal(total)).astype(np.float32) * 0.1     # non-negative: AdaGrad / RMSProp / AdaDelta / Adam v are sums of squares
    h2 = np.abs(rng.standard_normal(total)).astype(np.float32) * 0.1
    if kind in ("Nesterov", "Adam"):
        h = rng.standard_normal(total).astype(np.float32) * 0.1
    rates = [float(r) for r in rng.uniform(0.001, 0.05, len(counts))]
    decays = [float(d) for d in rng.uniform(0.0, 0.01, len(counts))]
    hp, gs, t = _hp(kind), 0.125, 3
    k_rates = [float(np.float32(r) * so.adam_correction(hp["momentum"], hp["momentum2"], t)) for r in rates] if kind == "Adam" else rates
    G, W, H = (torch.from_numpy(a.copy()).cuda() for a in (g, w, h))
    H2buf = torch.from_numpy(np.concatenate([np.zeros(h2_shift, np.float32), h2])).cuda()
    H2 = H2buf[h2_shift:] if kind in so.TWO_HISTORIES else None
    capi.solver_update_arena(kind, offsets, counts, k_rates, decays, G, W, H, H2, momentum=hp["momentum"], delta=hp["delta"],
                             rms_decay=hp["rms_decay"], beta1=hp["momentum"], beta2=hp["momentum2"], l2=l2, grad_scale=gs,
                             clear_grads=clear)
    torch.cuda.synchronize()
    got = [G.cpu().numpy(), W.cpu().numpy(), H.cpu().numpy(), H2.cpu().numpy() if H2 is not None else None]
    want = [g.copy(), w.copy(), h.copy(), h2.copy()]
    for s, (o, c) in enumerate(zip(offsets, counts)):
        sl = slice(o, o + c)
        out = so.update(kind, g[sl], w[sl], h[sl], h2[sl], hp, rates[s], decays[s], t=t, l2=l2, grad_scale=gs, clear_grads=clear)
        for k in range(4):
            if out[k] is not None:
                want[k][sl] = out[k]
    for k, name in enumerate(("g", "w", "h", "h2")):
        if got[k] is None:
            continue
        np.testing.assert_allclose(got[k], want[k], rtol=2e-5, atol=2e-6, err_msg=f"{kind} {name}")
    # elements outside every segment are bitwise untouched
    mask = np.ones(total, bool)
    for o, c in zip(offsets, counts):
        mask[o:o + c] = False
    assert np.array_equal(got[1][mask].view(np.uint32), w[mask].view(np.uint32))
    assert np.array_equal(got[0][mask].view(np.uint32), g[mask].view(np.uint32))


def test_sgd_kind_is_the_sgd_entry_bit_for_bit():
    import torch
    rng = np.random.default_rng(5)
    offsets, counts, total = _layout(rng)
    rates, decays = [0.01] * len(counts), [5e-4] * len(counts)
    a = [torch.from_numpy(rng.standard_normal(total).astype(np.float32)).cuda() for _ in range(3)]
    b = [x.clone() for x in a]
    capi.sgd_update_arena(offsets, counts, rates, decays, *a, 0.9, grad_scale=0.125)
    capi.solver_update_arena("SGD", offsets, counts, rates, decays, *b, momentum=0.9, grad_scale=0.125)
    torch.cuda.synchronize()
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))


@pytest.mark.parametrize("kind", NEW_KINDS)
def test_typed_solver_handle_four_iterations(kind):
    """4 iterations of a typed SGDSolver handle (lr policy "step", per-blob lr_mult / decay_mult, L1) against the oracle.  A blob with
    lr_mult = decay_mult = 0 and a zero diff goes through the kernel here (the handle marks no blob statistic) and must stay bitwise
    unchanged, histories included: that the update is the identity for such a blob is what lets ApplyUpdate leave BatchNorm
    statistics out of the launch."""
    rng = np.random.default_rng(11)
    counts = [37, 1000, 6, 4099, 12]
    lr_mult, decay_mult = [1.0, 2.0, 0.0, 0.5, 1.0], [1.0, 0.0, 0.0, 1.0, 2.0]
    hp = _hp(kind)
    base_lr, wd = 0.02, 0.004
    s = host_api.SGDSolver(type=kind, base_lr=base_lr, lr_policy="step", gamma=0.5, stepsize=2, max_iter=100, momentum=hp["momentum"],
                           weight_decay=wd, regularization_type="L1", delta=hp["delta"], momentum2=hp["momentum2"],
                           rms_decay=hp["rms_decay"])
    s.set_params(counts, lr_mult, decay_mult)
    two = kind in so.TWO_HISTORIES
    w = [rng.standard_normal(c).astype(np.float32) for c in counts]
    hist = [np.zeros(c, np.float32) for c in counts]
    hist2 = [np.zeros(c, np.float32) for c in counts]
    for i in range(len(counts)):
        s.set(i, w[i])
    for it in range(4):
        lr = oracle.learning_rate("step", it, base_lr, gamma=0.5, stepsize=2)
        for i, c in enumerate(counts):
            g = np.zeros(c, np.float32) if lr_mult[i] == 0 else rng.standard_normal(c).astype(np.float32)
            s.set(i, g, diff=True)
            if lr_mult[i] == 0 and decay_mult[i] == 0:
                continue
            _, w[i], hist[i], h2 = so.update(kind, g, w[i], hist[i], hist2[i], hp, lr * lr_mult[i], wd * decay_mult[i], t=it + 1,
                                             l2=False)
            if two:
                hist2[i] = h2
        s.step()
        assert s.iter() == it + 1
        for i in range(len(counts)):
            np.testing.assert_allclose(s.get(i, 0), w[i], rtol=2e-5, atol=2e-6, err_msg=f"{kind} it {it} blob {i}")
            np.testing.assert_allclose(s.get(i, 2), hist[i], rtol=2e-5, atol=2e-6)
            if two:
                np.testing.assert_allclose(s.get(i, 3), hist2[i], rtol=2e-5, atol=2e-6)
    assert np.array_equal(s.get(2, 0).view(np.uint32), w[2].view(np.uint32))
    assert not s.get(2, 2).any() and (not two or not s.get(2, 3).any())
    if not two:
        with pytest.raises(host_api.HostError, match="no second history"):
            s.get(0, 3)


# ------------------------------------------------------------------------------------------------------------------- whole net
def solver_text(kind, base_lr):
    hp = _hp(kind)
    return ('type: "%s" base_lr: %g lr_policy: "fixed" momentum: %g momentum2: %g delta: %g rms_decay: %g weight_decay: 0.0005 '
            'max_iter: 100' % (kind, base_lr, hp["momentum"], hp["momentum2"], hp["delta"], hp["rms_decay"]))


def make_trainer(spec, solver, rng, classes=10):
    t = host_api.Trainer(no.to_prototxt(spec), solver, num_classes=classes)
    params = []
    for i, (_, pk, shp) in enumerate(no.param_shapes(spec)):
        p = (rng.standard_normal(shp) * np.sqrt(2.0 / np.prod(shp[1:]))).astype(np.float32) if pk == "w" else \
            rng.uniform(0.5, 1.5, shp).astype(np.float32) if pk == "scale" else rng.uniform(-0.2, 0.2, shp).astype(np.float32)
        t.set_param(i, p)
        params.append(p)
    data = rng.standard_normal(spec[0]["shape"]).astype(np.float32)
    label = rng.integers(0, classes, spec[0]["shape"][0]).astype(np.float32)
    t.set_blob("data", data)
    t.set_blob("label", label)
    return t, params, data, label


def rel(a, ref, floor=1e-20):
    return float(np.max(np.abs(a.reshape(-1) - ref.reshape(-1))) / max(np.max(np.abs(ref)), floor))


@pytest.mark.parametrize("kind,net,base_lr", [("Adam", "resnet", 0.001), ("AdaDelta", "resnet", 0.05), ("Nesterov", "resnet", 0.05),
                                              ("AdaGrad", "lenet", 0.001), ("RMSProp", "lenet", 0.001)])
def test_steps_match_net_oracle(kind, net, base_lr):
    """3 training steps through TrainNet against netoracle forward / backward + the solver oracle, at the 1e-3 bar of
    test_trainer_gpu.py::test_sgd_steps_match_oracle.  Adam, AdaGrad and RMSProp divide by the gradient's own magnitude, so any
    gradient well above delta moves its weight by about base_lr: a ReLU unit that sits on its boundary in one computation and
    not in the other turns a rounding-level difference into a step of that size.  Their rates are kept at 1e-3 so that the bar
    measures the update rather than such flips."""
    spec = no.mini_resnet() if net == "resnet" else no.lenet()
    t, params, data, label = make_trainer(spec, solver_text(kind, base_lr), np.random.default_rng(1701))
    hp, two = _hp(kind), kind in so.TWO_HISTORIES
    ref = [p.copy() for p in params]
    hist = [np.zeros(p.size, np.float32) for p in params]
    hist2 = [np.zeros(p.size, np.float32) for p in params]
    ref_losses, losses = [], []
    for it in range(3):
        loss, grads, _, _ = no.forward_backward(spec, ref, data, label)
        ref_losses.append(loss)
        for i, g in enumerate(grads):
            _, w, hist[i], h2 = so.update(kind, g, ref[i], hist[i], hist2[i], hp, base_lr, 0.0005, t=it + 1)
            ref[i] = w.reshape(ref[i].shape)
            if two:
                hist2[i] = h2
        t.step(1)
        losses.append(t.loss())
    np.testing.assert_allclose(losses, ref_losses, rtol=2e-3)
    hf = 1e-3 * max(float(np.max(np.abs(x))) for x in hist)
    h2f = 1e-3 * max(float(np.max(np.abs(x))) for x in hist2) if two else 0
    for i in range(len(ref)):
        assert rel(t.get_param(i, 0), ref[i]) <= 2e-3, (kind, i)
        assert rel(t.get_param(i, 2), hist[i], hf) <= 5e-3, (kind, i)
        if two:
            assert rel(t.get_param(i, 3), hist2[i], h2f) <= 5e-3, (kind, i)
        assert not t.get_param(i, 1).any()


def _num_history(state):
    L = host_api.lib()
    L.b2h_wire_load.restype = C.c_void_p
    h = L.b2h_wire_load(state.encode(), 1)
    assert h
    L.b2h_wire_num_history.argtypes = [C.c_void_p]
    L.b2h_wire_destroy.argtypes = [C.c_void_p]
    n = L.b2h_wire_num_history(h)
    L.b2h_wire_destroy(h)
    return n


@pytest.mark.parametrize("kind", ["Adam", "AdaDelta"])
def test_snapshot_restore_with_two_histories(kind, tmp_path):
    """step, snapshot, step  ==  fresh trainer, restore, step: bitwise, both histories included; the .solverstate holds 2 * np
    history blobs, [h_0 .. h_np-1, h2_0 .. h2_np-1] as AdamPreSolve lays them out."""
    spec = no.mini_resnet()
    solver = solver_text(kind, 0.001)
    t, _, data, label = make_trainer(spec, solver, np.random.default_rng(1701))
    t.step(2)
    state = t.snapshot(str(tmp_path / "snap"))
    t.step(2)
    want = [[t.get_param(i, k).copy() for i in range(t.num_params())] for k in (0, 2, 3)]
    t2, _, _, _ = make_trainer(spec, solver, np.random.default_rng(7))
    t2.set_blob("data", data)
    t2.set_blob("label", label)
    t2.restore(state)
    assert t2.iter() == 2
    t2.step(2)
    assert t2.loss() == t.loss()
    for k, what in enumerate((0, 2, 3)):
        for i in range(t.num_params()):
            assert np.array_equal(t2.get_param(i, what).view(np.uint32), want[k][i].view(np.uint32)), (what, i)
    assert _num_history(state) == 2 * t.num_learnable()
    # a one-history state does not restore into a two-history solver
    t3, _, _, _ = make_trainer(spec, SOLVER_SGD, np.random.default_rng(8))
    t3.step(1)
    sgd_state = t3.snapshot(str(tmp_path / "sgd"))
    with pytest.raises(host_api.HostError, match="Incorrect length of history blobs"):
        t2.restore(sgd_state)


SOLVER_SGD = 'base_lr: 0.01 lr_policy: "fixed" momentum: 0.9 weight_decay: 0.0005 max_iter: 100'


# ------------------------------------------------------------------------------------------------------------------- CLI
@pytest.mark.parametrize("solver,classes", [("examples/solvers/adam/solver.prototxt", 1000),
                                            ("examples/mnist/lenet_solver_rmsprop.prototxt", 10),
                                            ("examples/mnist/lenet_adadelta_solver.prototxt", 10)])
def test_cli_trains_reference_solver_files(solver, classes, tmp_path):
    """`caffe.py train` on the reference's own solver files (run from the fixture directory: their paths are relative to it), on the
    synthetic source: finite losses, and a .solverstate with np or 2 * np history blobs."""
    prefix = str(tmp_path / "snap")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "caffe.py"), "train", "--solver=" + solver, "--iterations=3",
                        "--batch=64", "--display=1", "--classes=%d" % classes, "--snapshot_prefix=" + prefix],
                       capture_output=True, text=True, cwd=REF, timeout=600, env=dict(os.environ, B2C_DATA="synthetic"))
    assert r.returncode == 0, r.stderr[-3000:]
    kind = host_api.solver_describe(host_api.open_solver(os.path.join(REF, solver))[0])["type"]
    assert "with %s:" % kind in r.stdout
    losses = [float(x) for x in re.findall(r"loss = (\S+)", r.stdout)]
    assert len(losses) == 3 and all(np.isfinite(losses)), r.stdout
    states = [f for f in os.listdir(tmp_path) if f.endswith(".solverstate")]
    assert states == ["snap_iter_3.solverstate"]
    # resume from the snapshot (--snapshot), then fine-tune from its weights (--weights)
    base = [sys.executable, os.path.join(ROOT, "tools", "caffe.py"), "train", "--solver=" + solver, "--iterations=2", "--batch=64",
            "--display=1", "--classes=%d" % classes]
    env = dict(os.environ, B2C_DATA="synthetic")
    r2 = subprocess.run(base + ["--snapshot=" + str(tmp_path / states[0]), "--snapshot_prefix=" + prefix], capture_output=True, text=True,
                        cwd=REF, timeout=600, env=env)
    assert r2.returncode == 0, r2.stderr[-3000:]
    assert "at iteration 3" in r2.stdout and "Iteration 5 (" in r2.stdout and os.path.exists(prefix + "_iter_5.solverstate")
    r3 = subprocess.run(base + ["--weights=" + prefix + "_iter_5.caffemodel", "--snapshot_prefix=" + str(tmp_path / "ft")],
                        capture_output=True, text=True, cwd=REF, timeout=600, env=env)
    assert r3.returncode == 0, r3.stderr[-3000:]
    assert "Finetuning from" in r3.stdout and os.path.exists(str(tmp_path / "ft_iter_2.solverstate"))
    assert all(np.isfinite([float(x) for x in re.findall(r"loss = (\S+)", r2.stdout + r3.stdout)]))
    n = _num_history(str(tmp_path / states[0]))
    nets = host_api.Net(os.path.join(REF, host_api.open_solver(os.path.join(REF, solver))[1]), "TRAIN", batch_override=1)
    np_ = len(nets.learnable_params())
    assert n == (2 * np_ if kind in so.TWO_HISTORIES else np_)


# ------------------------------------------------------------------------------------------------------------------- multi-GPU
@pytest.mark.parametrize("kind", ["Adam", "AdaDelta"])
def test_two_ranks_equal_one_rank(kind):
    """Two processes, one GPU each, through P2PSync / ReduceScheduler (tests/solver_rank_worker.py): parameters and both histories
    are bit-identical across ranks and equal one solver on the concatenated batch, within tests/test_multi_gpu.py's tolerances
    (1e-5 parameters, 1e-4 histories with a floor at 1e-3 of the largest)."""
    import socket
    import tempfile
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import multi_rank_worker as mw
    import solver_rank_worker as sw
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    global_batch, steps = 64, 3
    with tempfile.TemporaryDirectory() as td:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
               "--master-port", str(port), os.path.join(ROOT, "tests", "solver_rank_worker.py"), td, kind, str(global_batch), str(steps)]
        r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-4000:])
        ranks = [dict(np.load(os.path.join(td, f"rank{i}.npz"))) for i in range(2)]
    params, data, label = mw.build_case(global_batch)
    one = sw.run(kind, global_batch, params, data, label, steps)
    for key in ("p", "h", "g"):
        floor = 0.0 if key == "p" else 1e-3 * max(float(np.abs(one[f"{key}{j}"]).max()) for j in range(len(params)))
        for i in range(len(params)):
            a, b = ranks[0][f"{key}{i}"], ranks[1][f"{key}{i}"]
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), f"{key}{i} differs across ranks"
            assert rel(a, one[f"{key}{i}"], max(floor, 1e-20)) < (1e-5 if key == "p" else 1e-4), (key, i)

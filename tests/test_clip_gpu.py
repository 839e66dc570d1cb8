"""clip_gradients on the GPU: the norm's partials (b2c_arena_sumsq), the factor (b2c_clip_factor) and the scaled update
(b2c_solver_update_arena_scaled) against the float64 clip oracle (tests/clip_oracle.py) and the unscaled update, then TrainNet and
`caffe.py train` with solver files that set the field.  Every kernel case asserts its launch plan first, runs twice for identical
bits, and keeps NaN sentinels in the gaps between segments: their bits must survive and they must not reach the norm."""
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from caffe_mpi_b200 import capi, host_api
import clip_oracle as co
import netoracle as no
import solver_oracle as so
from test_solvers_gpu import _hp, make_trainer, rel, solver_text

pytestmark = pytest.mark.gpu
F = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "tests", "golden", "reference_models")
RESNET50 = os.path.join(REF, "models", "resnet50", "train_val.prototxt")


def bits(t):
    return t.detach().cpu().numpy().view(np.uint8).copy()


def layout(counts, start=3):
    """offsets with 0-2 float gaps after each segment (odd start: the segments peel heads), and the arena length"""
    offs, off = [], start
    for k, c in enumerate(counts):
        offs.append(off)
        off += c + (k % 3)
    return offs, off + 2


def put(counts, offs, total, gen):
    """a float32 arena of NaN sentinels with gen(count) written at each segment"""
    a = np.full(total, np.nan, F)
    for o, c in zip(offs, counts):
        a[o:o + c] = gen(c)
    return a


def segs_of(a, counts, offs):
    return [a[o:o + c] for o, c in zip(offs, counts)]


def run_norm(g, counts, offs, clip, s_n=1.0):
    """partials, (norm, factor, clipped) and the state tensor; asserts the plan and that a second run gives the same bits"""
    import torch
    slots, npart = host_api.clip_slots(counts)
    q = capi.sumsq_plan(offs, counts, slots, g.data_ptr())
    assert q["npartials"] == npart
    nonempty = sum(1 for c in counts if c)
    assert [n for n, _ in q["launches"]] == [min(96, nonempty - 96 * i) for i in range(-(-nonempty // 96))]
    for s, c in enumerate(counts):
        assert q["segs"][s]["blocks"] == -(-c // 4096) and q["segs"][s]["slot"] == slots[s] and q["segs"][s]["vec"] == (1 if c else 0)
    out = []
    for _ in range(2):
        P = torch.full((max(npart, 1),), float("nan"), dtype=torch.float64, device="cuda")
        st = torch.zeros(4, dtype=torch.float32, device="cuda")
        capi.arena_sumsq(offs, counts, slots, g, P)
        capi.clip_factor(P, npart, s_n, clip, st)
        torch.cuda.synchronize()
        out.append((P[:npart].cpu().numpy(), capi.clip_state(st), st))
    assert np.array_equal(out[0][0].view(np.uint64), out[1][0].view(np.uint64)) and out[0][1] == out[1][1]
    return out[0][0], out[0][1], out[0][2], slots


def block_sums(a, counts, offs, slots, npart):
    """math.fsum of each block's squares, at its slot"""
    want = np.zeros(npart)
    for o, c, s in zip(offs, counts, slots):
        for b in range(-(-c // 4096)):
            x = a[o + 4096 * b:o + min(c, 4096 * (b + 1))].astype(np.float64)
            want[s + b] = math.fsum((x * x).tolist())
    return want


def ulps(a, b):
    return abs(int(np.float32(a).view(np.int32)) - int(np.float32(b).view(np.int32)))


def _counts(rng, n):
    c = [int(x) for x in rng.integers(1, 300, n)] + [40000, 7, 0, 4097, 4096, 1]
    return c


@pytest.mark.parametrize("nseg", [1, 97, 193])
def test_norm_is_exact_on_dyadic_data(nseg):
    """k/64 with |k| <= 64: every square and every partial sum is exact in double, so each partial equals the exact block sum and the
    norm equals the oracle's float exactly"""
    import torch
    rng = np.random.default_rng(nseg)
    counts = _counts(rng, nseg)
    offs, total = layout(counts)
    a = put(counts, offs, total, lambda c: rng.integers(-64, 65, c).astype(F) / F(64))
    g = torch.from_numpy(a).cuda()
    before = bits(g)
    P, (norm, factor, clipped), _, slots = run_norm(g, counts, offs, 1.0)
    assert np.array_equal(bits(g), before)
    assert np.array_equal(P, block_sums(a, counts, offs, slots, len(P)))
    want_norm, want_factor = co.clip_factor(segs_of(a, counts, offs), 1.0)
    assert F(norm) == want_norm and F(factor) == want_factor and clipped == 1


@pytest.mark.parametrize("s_n", [1.0, 0.5, 1 / 3])
def test_norm_within_one_ulp_on_wide_data(s_n):
    import torch
    rng = np.random.default_rng(7)
    counts = _counts(rng, 130)
    offs, total = layout(counts)
    a = put(counts, offs, total, lambda c: (rng.standard_normal(c) * np.exp2(rng.integers(-30, 30, c))).astype(F))
    g = torch.from_numpy(a).cuda()
    P, (norm, factor, _), _, slots = run_norm(g, counts, offs, 1e30, s_n)
    want = block_sums(a, counts, offs, slots, len(P))
    assert np.all(np.abs(P - want) <= 4096 * 2.0 ** -53 * want)
    want_norm, want_factor = co.clip_factor(segs_of(a, counts, offs), 1e30, s_n)
    assert ulps(norm, want_norm) <= 1 and factor == 1.0


def _update_arrays(rng, kind, counts, offs, total):
    g = put(counts, offs, total, lambda c: (rng.standard_normal(c) * 1e-2).astype(F))
    w = put(counts, offs, total, lambda c: (rng.standard_normal(c) * 0.05).astype(F))
    pos = kind not in ("SGD", "Nesterov", "Adam")
    h = put(counts, offs, total, lambda c: ((np.abs if pos else np.asarray)(rng.standard_normal(c)) * 1e-3).astype(F))
    h2 = put(counts, offs, total, lambda c: (np.abs(rng.standard_normal(c)) * 1e-6).astype(F))
    return g, w, h, h2


@pytest.mark.parametrize("clipped", [False, True], ids=["unclipped", "clipped"])
@pytest.mark.parametrize("kind", so.KINDS)
def test_scaled_update_is_the_unscaled_update_at_the_clipped_grad_scale(kind, clipped):
    """the unclipped case equals b2c_solver_update_arena at the original grad_scale; the clipped one at fl(grad_scale * factor) with
    the factor read back from the device; both bit for bit, gaps included"""
    import torch
    rng = np.random.default_rng(11 + so.KINDS.index(kind))
    counts = _counts(rng, 130)
    offs, total = layout(counts)
    arrays = _update_arrays(rng, kind, counts, offs, total)
    s_n, gs = 0.5, float(F(F(1) / F(2) / F(1) / F(2)))             # two solvers, iter_size 2
    want_norm, _ = co.clip_factor(segs_of(arrays[0], counts, offs), 1e30, s_n)
    clip = float(want_norm) * (0.25 if clipped else 4.0)
    G = torch.from_numpy(arrays[0]).cuda()
    _, (norm, factor, nclip), st, _ = run_norm(G, counts, offs, clip, s_n)
    assert ulps(norm, want_norm) <= 1 and nclip == int(clipped)
    assert (F(factor) == F(clip) / F(norm)) if clipped else factor == 1.0
    rates = [float(F(0.01 * (1 + s / 100))) for s in range(len(counts))]
    decays = [float(F(5e-4 * (1 + s / 100))) for s in range(len(counts))]
    hp = dict(momentum=0.0 if kind in ("AdaGrad", "RMSProp") else 0.9, delta=1e-8, rms_decay=0.95, beta1=0.9, beta2=0.999)
    two = kind in so.TWO_HISTORIES
    outs = []
    for scaled in (True, True, False):
        g, w, h, h2 = (torch.from_numpy(x.copy()).cuda() for x in arrays)
        if scaled:
            capi.solver_update_arena_scaled(kind, offs, counts, rates, decays, g, w, h, h2 if two else None, factor=st[1:2], grad_scale=gs, **hp)
        else:
            capi.solver_update_arena(kind, offs, counts, rates, decays, g, w, h, h2 if two else None, grad_scale=float(F(F(gs) * F(factor))),
                                     **hp)
        torch.cuda.synchronize()
        outs.append([bits(x) for x in (g, w, h, h2)])
    for k in range(4):
        assert np.array_equal(outs[0][k], outs[1][k]) and np.array_equal(outs[0][k], outs[2][k]), (kind, k)
    gaps = np.isnan(arrays[1])
    assert np.isnan(outs[0][1].view(F)[gaps]).all() and np.array_equal(outs[0][1].view(np.uint32)[gaps], arrays[1].view(np.uint32)[gaps])


def test_zero_gradient_and_clip_zero():
    import torch
    counts = [5, 4097, 300]
    offs, total = layout(counts)
    z = torch.from_numpy(put(counts, offs, total, lambda c: np.zeros(c, F))).cuda()
    _, (norm, factor, n), _, _ = run_norm(z, counts, offs, 0.0)
    assert (norm, factor, n) == (0.0, 1.0, 0)                   # 0 > 0 is false
    rng = np.random.default_rng(5)
    arrays = _update_arrays(rng, "SGD", counts, offs, total)
    G = torch.from_numpy(arrays[0]).cuda()
    _, (norm, factor, n), st, _ = run_norm(G, counts, offs, 0.0)
    assert norm > 0 and factor == 0.0 and n == 1
    outs = []
    for scaled in (True, False):
        g, w, h, _ = (torch.from_numpy(x.copy()).cuda() for x in arrays)
        rates, decays = [0.01] * 3, [5e-4] * 3
        if scaled:
            capi.solver_update_arena_scaled("SGD", offs, counts, rates, decays, g, w, h, factor=st[1:2], momentum=0.9)
        else:
            capi.solver_update_arena("SGD", offs, counts, rates, decays, g, w, h, momentum=0.9, grad_scale=0.0)
        torch.cuda.synchronize()
        outs.append([bits(x) for x in (g, w, h)])
    assert all(np.array_equal(a, b) for a, b in zip(*outs))


def test_one_segment_of_2_26_plus_3():
    import torch
    c = (1 << 26) + 3
    rng = np.random.default_rng(9)
    k = rng.integers(-64, 65, c).astype(np.int64)
    a = np.full(c + 8, np.nan, F)
    a[3:3 + c] = k.astype(F) / F(64)
    g = torch.from_numpy(a).cuda()
    _, (norm, _, _), _, _ = run_norm(g, [c], [3], 1e30)
    exact = float(int((k * k).sum())) / 4096.0                  # every partial exact: the integer sum
    assert F(norm) == F(math.sqrt(exact))


def test_resnet50_arena():
    """ResNet-50's 161 learnable segments with realistic gradient magnitudes: norm within 1 ulp, and the scaled SGD update equals the
    unscaled one at fl(grad_scale * factor)"""
    import torch
    lp = host_api.Net(open(RESNET50).read(), is_text=True).learnable_params()
    counts = [c for _, c, _, _ in lp]
    offs, off = [], 0
    for c in counts:
        offs.append(off)
        off += c + (c & 1)
    rng = np.random.default_rng(31)
    a = (rng.standard_normal(off) * 1e-3).astype(F)
    G = torch.from_numpy(a).cuda()
    want_norm, _ = co.clip_factor(segs_of(a, counts, offs), 1e30)
    _, (norm, factor, _), st, _ = run_norm(G, counts, offs, float(want_norm) / 2)
    assert ulps(norm, want_norm) <= 1 and F(factor) == F(F(want_norm) / 2) / F(norm)
    w0 = (rng.standard_normal(off) * 0.05).astype(F)
    outs = []
    for scaled in (True, False):
        g, w, h = G.clone(), torch.from_numpy(w0).cuda(), torch.zeros(off, device="cuda")
        rates, decays = [0.1] * len(counts), [1e-4] * len(counts)
        if scaled:
            capi.solver_update_arena_scaled("SGD", offs, counts, rates, decays, g, w, h, factor=st[1:2], momentum=0.9)
        else:
            capi.solver_update_arena("SGD", offs, counts, rates, decays, g, w, h, momentum=0.9, grad_scale=float(factor))
        torch.cuda.synchronize()
        outs.append([bits(x) for x in (w, h)])
    assert all(np.array_equal(x, y) for x, y in zip(*outs))


# ------------------------------------------------------------------------------------------------------------------- TrainNet
def _solver(kind, base_lr, clip):
    return solver_text(kind, base_lr) + " clip_gradients: %r" % clip


@pytest.mark.parametrize("kind,base_lr", [("SGD", 0.05), ("Adam", 0.001)])
def test_trainer_steps_match_net_oracle(kind, base_lr):
    """3 clipped steps of the mini ResNet through TrainNet against netoracle + the clip oracle + the solver oracle, at
    test_solvers_gpu.py's tolerances; the clip is set between the first and the last step's norm so that some steps clip"""
    spec = no.mini_resnet()
    hp = _hp(kind)
    _, params, data, label = make_trainer(spec, solver_text(kind, base_lr), np.random.default_rng(1701))
    norms = co.replay(kind, spec, params, data, label, 3, base_lr, 1e30, hp)[4]
    clip = float(np.median(norms)) * 1.001                   # the median step's norm stays clear of the clip
    t, params, data, label = make_trainer(spec, _solver(kind, base_lr, clip), np.random.default_rng(1701))
    ref_losses, ref, hist, hist2, ref_norms = co.replay(kind, spec, params, data, label, 3, base_lr, clip, hp)
    losses, got_norms = [], []
    for _ in range(3):
        t.step(1)
        losses.append(t.loss())
        got_norms.append(t.clip_state()[0])
    np.testing.assert_allclose(losses, ref_losses, rtol=2e-3)
    np.testing.assert_allclose(got_norms, ref_norms, rtol=2e-3)
    assert t.clip_state()[2] == sum(1 for n in ref_norms if n > F(clip)) and 0 < t.clip_state()[2] < 3
    hf = 1e-3 * max(float(np.max(np.abs(x))) for x in hist)
    for i in range(len(ref)):
        assert rel(t.get_param(i, 0), ref[i]) <= 2e-3, (kind, i)
        assert rel(t.get_param(i, 2), hist[i], hf) <= 5e-3, (kind, i)
        assert not t.get_param(i, 1).any()


@pytest.mark.parametrize("kind", ["SGD", "Adam"])
def test_huge_clip_is_bitwise_the_unclipped_trainer(kind):
    spec = no.mini_resnet()
    a, params, _, _ = make_trainer(spec, solver_text(kind, 0.01), np.random.default_rng(3))
    b, _, _, _ = make_trainer(spec, _solver(kind, 0.01, 1e30), np.random.default_rng(3))
    for t in (a, b):
        t.step(3)
        t.sync()
    assert b.clip_state()[1:] == (1.0, 0)
    for i in range(len(params)):
        for what in (0, 2):
            assert np.array_equal(a.get_param(i, what).view(np.uint32), b.get_param(i, what).view(np.uint32)), (i, what)


def test_two_gpus_equal_one():
    """two processes, one GPU each, through P2PSync: ranks bit-identical, within 1e-5 of one solver on the concatenated batch"""
    import socket
    import tempfile
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import clip_rank_worker as cw
    import multi_rank_worker as mw
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    global_batch, steps = 64, 3
    with tempfile.TemporaryDirectory() as td:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
               "--master-port", str(port), os.path.join(ROOT, "tests", "clip_rank_worker.py"), td, str(global_batch), str(steps)]
        r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-4000:])
        ranks = [dict(np.load(os.path.join(td, f"rank{i}.npz"))) for i in range(2)]
    params, data, label = mw.build_case(global_batch)
    one = cw.run(global_batch, params, data, label, steps)
    assert 0 < one["clipped"] and ranks[0]["clipped"] == ranks[1]["clipped"] == one["clipped"]
    for key in ("p", "h"):
        floor = 0.0 if key == "p" else 1e-3 * max(float(np.abs(one[f"{key}{j}"]).max()) for j in range(len(params)))
        for i in range(len(params)):
            a, b = ranks[0][f"{key}{i}"], ranks[1][f"{key}{i}"]
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), f"{key}{i} differs across ranks"
            assert rel(a, one[f"{key}{i}"], max(floor, 1e-20)) < (1e-5 if key == "p" else 1e-4), (key, i)


# ------------------------------------------------------------------------------------------------------------------- CLI
def test_cli_trains_lenet_with_clip_gradients(tmp_path):
    """`caffe.py train` on the reference's lenet_solver.prototxt plus clip_gradients, from an LMDB of synthetic digits: it trains,
    the loss falls, stderr carries the reference's clipping line at display points, and stdout has the same lines as without
    clipping"""
    from caffe_mpi_b200 import lmdb_io
    rng = np.random.default_rng(2)
    db = str(tmp_path / "train_lmdb")
    protos = np.clip(rng.normal(128, 60, (10, 1, 28, 28)), 0, 255)
    labels = rng.integers(0, 10, 640)
    imgs = np.clip(protos[labels] + rng.normal(0, 20, (640, 1, 28, 28)), 0, 255).astype(np.uint8)
    lmdb_io.write_datum_lmdb(db, imgs, labels)
    net = open(os.path.join(REF, "examples", "mnist", "lenet_train_test.prototxt")).read()
    net = re.sub(r'source: "[^"]*_lmdb"', 'source: "%s"' % db, net)
    (tmp_path / "net.prototxt").write_text(net)
    solver = open(os.path.join(REF, "examples", "mnist", "lenet_solver.prototxt")).read()
    solver = re.sub(r'net: "[^"]*"', 'net: "%s"' % (tmp_path / "net.prototxt"), solver)
    solver = re.sub(r"(test_iter|test_interval|snapshot|snapshot_prefix): \S+", "", solver)
    outs = {}
    for name, extra in (("clip", "clip_gradients: 1\n"), ("plain", "")):
        path = tmp_path / (name + ".prototxt")
        path.write_text(solver + extra)
        r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "caffe.py"), "train", "--solver=" + str(path), "--iterations=60",
                            "--display=20"], capture_output=True, text=True, cwd=str(tmp_path), timeout=600,
                           env=dict(os.environ, B2C_DATA="db"))
        assert r.returncode == 0, r.stderr[-3000:]
        outs[name] = r
    losses = [float(x) for x in re.findall(r"loss = (\S+)", outs["clip"].stdout)]
    assert len(losses) == 3 and all(np.isfinite(losses)) and losses[-1] < losses[0], outs["clip"].stdout
    lines = re.findall(r"Gradient clipping: scaling down gradients \(L2 norm (\S+) > 1\) by scale factor (\S+)", outs["clip"].stderr)
    assert lines, outs["clip"].stderr[-2000:]
    for n, f in lines:
        assert float(n) > 1 and abs(float(f) - 1 / float(n)) < 1e-4
    assert "Gradient clipping" not in outs["clip"].stdout + outs["plain"].stderr
    strip = lambda s: [re.sub(r"^I\d+ [\d:]+ |\(.*?iter/s.*?\)|loss = \S+", "", ln) for ln in s.splitlines()]
    assert strip(outs["clip"].stdout) == strip(outs["plain"].stdout)

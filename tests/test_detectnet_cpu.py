"""The parts of NVCaffe's DetectNet example that are built here, on the CPU: the L1Loss float64 form against finite differences
and its Net shapes and messages; Data layers over float_data datums (DIGITS' label databases) through the DataReader and the
product DataLayer on the stream-order simulator; and an image and a label database read side by side -- by the readers, by two
Data layers in one TrainNet, and by two solvers -- delivering the same records in every batch."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import detectnet_oracle as dno
from caffe_mpi_b200 import capi, data_api, lmdb_io
from test_data_cpu import oracle_batches

HERE = os.path.dirname(os.path.abspath(__file__))
SOLVER = 'base_lr: 0.05 lr_policy: "fixed" momentum: 0.9 max_iter: 100 solver_mode: GPU'


def _fd(f, x, eps=1e-6):
    g = np.zeros_like(x)
    for i in np.ndindex(x.shape):
        xp, xm = x.copy(), x.copy()
        xp[i] += eps
        xm[i] -= eps
        g[i] = (f(xp) - f(xm)) / (2 * eps)
    return g


# ---------------------------------------------------------------------------------------------------- L1Loss
def test_l1_loss_known_answer_and_gradients():
    """loss = sum |a - b| / num; gradients +-loss_weight / num * sign(a - b), by finite differences away from the kinks."""
    a = np.array([[1.0, -2.0, 0.5], [3.0, 0.0, -1.0]])
    b = np.array([[0.0, 1.0, 0.5], [1.0, -4.0, 2.0]])
    loss, d = dno.l1_loss(a, b)
    assert loss == (1 + 3 + 0 + 2 + 4 + 3) / 2
    ga, gb = dno.l1_backward(d, 2, loss_weight=2.0)
    assert np.array_equal(ga, [[1.0, -1.0, 0.0], [1.0, 1.0, -1.0]]) and np.array_equal(gb, -ga)
    rng = np.random.default_rng(0)
    a, b = rng.standard_normal((3, 4)), rng.standard_normal((3, 4))
    _, d = dno.l1_loss(a, b)
    ga, gb = dno.l1_backward(d, 3, loss_weight=2.0)
    assert np.allclose(ga, _fd(lambda z: 2.0 * dno.l1_loss(z, b)[0], a), atol=1e-7)
    assert np.allclose(gb, _fd(lambda z: 2.0 * dno.l1_loss(a, z)[0], b), atol=1e-7)


def test_l1_loss_f32_restatement_and_sign_rule():
    a = np.array([0.5, -0.25, 3.0, 1.0], np.float32)
    b = np.array([0.25, -0.25, -1.0, 2.0], np.float32)
    loss, d = dno.l1_loss_f32(a, b, 2)
    assert loss == np.float32(5.25 / 2) and np.array_equal(d, a - b)
    g = dno.l1_backward_f32(d, -0.5)
    assert np.array_equal(g, [-0.5, 0.0, -0.5, 0.5]) and not np.signbit(g[1])      # sign(0) = 0, written as +0


def _net(text):
    from caffe_mpi_b200 import host_api as h
    return h.Net(text, "TRAIN", is_text=True)


_IN = ('layer { name: "x" type: "Input" top: "a" top: "b" top: "c" top: "d" input_param { shape { dim: 2 dim: 3 dim: 4 } '
       'shape { dim: 2 dim: 12 } shape { dim: 2 dim: 5 } shape { dim: 3 dim: 12 } } }\n')


def test_l1_loss_in_the_graph():
    n = _net("force_backward: true\n" + _IN + 'layer { name: "l" type: "L1Loss" bottom: "a" bottom: "b" top: "l" loss_weight: 2 }\n')
    assert n.loss_blob() == "l"
    assert [l[1:] for l in n.layers()][-1] == ("L1Loss", ())
    assert n.backward_plan()[-1] == (True, [True, True])               # both bottoms take a gradient (AllowForceBackward)


@pytest.mark.parametrize("bottoms,msg", [('bottom: "a" bottom: "c"', "Inputs must have the same dimension."),
                                         ('bottom: "b" bottom: "d"', "The data and label should have the same number.")])
def test_l1_loss_shape_errors(bottoms, msg):
    from caffe_mpi_b200 import host_api as h
    with pytest.raises(h.HostError, match=msg):
        _net(_IN + 'layer { name: "l" type: "L1Loss" %s top: "l" }\n' % bottoms)


# ---------------------------------------------------------------------------------------------------- float_data datums
def write_float_lmdb(path, arrays, labels=None):
    """One float_data Datum (no `data`) per [C][H][W] array, under convert_imageset's keys, as DIGITS writes label databases."""
    items = []
    for i, a in enumerate(arrays):
        c, h, w = a.shape
        items.append((lmdb_io.caffe_key(i), data_api.datum_serialize(c, h, w, b"", 0 if labels is None else int(labels[i]),
                                                                        float_data=[float(v) for v in a.reshape(-1)])))
    lmdb_io.write_lmdb(path, items)
    return path


def label_arrays(n, max_boxes, seed=0):
    """n DIGITS-layout label arrays; image i holds i % (max_boxes + 1) boxes, so each record is recognisable."""
    rng = np.random.default_rng(seed)
    return np.stack([dno.label_datum(dno.random_boxes(rng, i % (max_boxes + 1), 1248, 384), max_boxes) for i in range(n)])


def test_label_datum_layout():
    lab = label_arrays(4, 3)
    assert lab.shape == (4, 1, 4, 16) and lab.dtype == np.float32
    assert [tuple(l[0, 0, :2]) for l in lab] == [(0, 16), (1, 16), (2, 16), (3, 16)]
    assert not lab[1, 0, 2:].any() and lab[1, 0, 1].any()


@pytest.mark.parametrize("P,S,rank", [(1, 1, 0), (2, 1, 0), (3, 2, 1), (2, 3, 2)])
def test_float_datum_reader_delivers_the_values_verbatim(tmp_path, P, S, rank):
    n, B = 29, 4
    lab = label_arrays(n, 5)
    write_float_lmdb(str(tmp_path / "labels"), lab[:, 0][:, None])
    r = data_api.DataReader(str(tmp_path / "labels"), B, solver_count=S, solver_rank=rank, parser_threads=P)
    assert r.shape == (1, 6, 16) and r.dtype == np.float32
    for i, want in enumerate(oracle_batches(n, 9, B, S, rank, P)):
        data, _, ids, bid = r.next()
        assert bid == i and list(ids) == [rec for _, rec in want]
        assert np.array_equal(data.view(np.uint32), lab[[p for p, _ in want]].view(np.uint32)), f"batch {i}"
    r.close()


@pytest.mark.parametrize("P", [1, 2, 3])
@pytest.mark.parametrize("S,rank", [(1, 0), (2, 0), (2, 1), (4, 3)])
def test_image_and_label_readers_hold_the_same_records(tmp_path, P, S, rank):
    """Two readers with one batch size and one parser count, over an image and a label database of the same length: batch i of
    each holds the same record positions for every rank.  With several solvers and DIFFERENT parser counts the partition would
    pair different records -- which is why TrainNet gives a net's database layers one count."""
    n, B = 37, 3
    rng = np.random.default_rng(P * 10 + S + rank)
    imgs = rng.integers(0, 256, (n, 3, 4, 6), dtype=np.uint8)
    imgs[:, 0, 0, 0] = np.arange(n)                                     # the record's index, in the image
    lmdb_io.write_datum_lmdb(str(tmp_path / "img"), imgs, np.zeros(n, np.int64))
    lab = label_arrays(n, 2, seed=P)
    lab[:, 0, 0, 2] = np.arange(n)                                      # and in the label's header row (a spare column)
    write_float_lmdb(str(tmp_path / "lab"), lab)
    ri = data_api.DataReader(str(tmp_path / "img"), B, solver_count=S, solver_rank=rank, parser_threads=P)
    rl = data_api.DataReader(str(tmp_path / "lab"), B, solver_count=S, solver_rank=rank, parser_threads=P)
    for _ in range(2 * n // B):
        di, _, ii, _ = ri.next()
        dl, _, il, _ = rl.next()
        assert np.array_equal(ii, il)
        assert np.array_equal(di[:, 0, 0, 0].astype(np.float32), dl[:, 0, 0, 2])
    ri.close()
    rl.close()
    if S > 1 and P > 1:
        recs = lambda p: [[q for q, _ in b] for b in oracle_batches(n, 4, B, S, rank, p)]
        assert recs(P) != recs(1)


def test_float_and_uint8_datums_do_not_mix(tmp_path):
    items = [(lmdb_io.caffe_key(0), data_api.datum_serialize(1, 1, 2, b"", 0, float_data=[1.0, 2.0])),
             (lmdb_io.caffe_key(1), lmdb_io.datum_bytes(np.zeros((1, 1, 2), np.uint8), 0))]
    lmdb_io.write_lmdb(str(tmp_path / "mixed"), items)
    r = data_api.DataReader(str(tmp_path / "mixed"), 2)
    with pytest.raises(data_api.DataError, match="mixes float_data datums and uint8 datums"):
        r.next()
    r.close()
    bad = [(lmdb_io.caffe_key(0), data_api.datum_serialize(1, 2, 2, b"", 0, float_data=[1.0, 2.0]))]
    lmdb_io.write_lmdb(str(tmp_path / "short"), bad)
    with pytest.raises(data_api.DataError, match="float_data size disagrees"):
        data_api.DataReader(str(tmp_path / "short"), 1)


# ---- the product DataLayer over float datums, on the stream-order model ---------------------------------------------------------------
@pytest.fixture(scope="module")
def sim():
    capi.lib()
    r = subprocess.run(["make", "-C", os.path.join(HERE, "sim")], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.fail("tests/sim does not build:\n" + r.stdout[-2000:] + r.stderr[-4000:])
    L = C.CDLL(os.path.join(HERE, "sim", "libdatasim.so"))
    L.sim_last_error.restype = C.c_char_p
    L.sim_create.restype = C.c_void_p
    L.sim_create.argtypes = [C.c_char_p, C.c_ulonglong, C.c_int, C.c_int]
    L.sim_destroy.argtypes = [C.c_void_p]
    L.sim_shape.argtypes = [C.c_void_p, C.POINTER(C.c_int)]
    L.sim_load_batch.argtypes = [C.c_void_p]
    L.sim_read.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.fakecuda_set_eager.argtypes = [C.c_void_p, C.c_int]
    L.fakecuda_set_all_eager.argtypes = [C.c_int]
    return L


NET = ('name: "sim" layer {{ name: "label" type: "Data" top: "label" top: "unused" data_param {{ source: "{src}" backend: LMDB '
       'batch_size: {B} {dp} }} {tp} }}')


@pytest.mark.parametrize("compute_eager,copy_eager", [(0, 0), (1, 1), (0, 1), (1, 0)])
@pytest.mark.parametrize("P,S,rank", [(1, 1, 0), (3, 2, 1)])
def test_data_layer_copies_float_datums_verbatim_under_extreme_stream_orders(sim, tmp_path, monkeypatch, compute_eager, copy_eager, P, S, rank):
    monkeypatch.delenv("B2C_DATA", raising=False)
    L = sim
    n, B, steps = 23, 4, 11
    lab = label_arrays(n, 4, seed=7)
    path = write_float_lmdb(str(tmp_path / "labels"), lab, labels=np.arange(n) % 5)
    L.fakecuda_set_all_eager(0)
    h = L.sim_create(NET.format(src=path, B=B, dp="parser_threads: %d" % P, tp="").encode(), 1, S, rank)
    assert h, L.sim_last_error().decode()
    L.fakecuda_set_all_eager(copy_eager)
    L.fakecuda_set_eager(None, compute_eager)
    shp = (C.c_int * 4)()
    L.sim_shape(h, shp)
    assert tuple(shp) == (B, 1, 5, 16)
    got, lb = np.empty((B, 1, 5, 16), np.float32), np.empty(B, np.float32)
    want = oracle_batches(n, steps, B, S, rank, P)
    for i in range(steps):
        assert L.sim_load_batch(h) == 0, L.sim_last_error().decode()
        if i % 4 != 3 and i != steps - 1:
            continue
        assert L.sim_read(h, got.ctypes.data_as(C.c_void_p), lb.ctypes.data_as(C.c_void_p)) == 0, L.sim_last_error().decode()
        pos = [p for p, _ in want[i]]
        assert np.array_equal(got.view(np.uint32), lab[pos].view(np.uint32)), f"batch {i}"
        assert np.array_equal(lb, (np.array(pos) % 5).astype(np.float32))
    L.sim_destroy(h)
    L.fakecuda_set_all_eager(0)


@pytest.mark.parametrize("tp", ["crop_size: 2", "mirror: true", "scale: 0.5", "mean_value: 1"])
def test_float_datums_refuse_a_transform(sim, tmp_path, monkeypatch, tp):
    monkeypatch.delenv("B2C_DATA", raising=False)
    path = write_float_lmdb(str(tmp_path / "labels"), label_arrays(3, 1))
    h = sim.sim_create(NET.format(src=path, B=2, dp="", tp="transform_param { %s }" % tp).encode(), 1, 1, 0)
    assert not h
    assert "float_data, which are copied as they are: transform_param" in sim.sim_last_error().decode()
    ok = sim.sim_create(NET.format(src=path, B=2, dp="", tp="transform_param { scale: 1 mirror: false }").encode(), 1, 1, 0)
    assert ok, sim.sim_last_error().decode()
    sim.sim_destroy(ok)


# ---- two database Data layers in one TrainNet, one and two solvers (libtrainsim.so) ----------------------------------------------------
@pytest.fixture(scope="module")
def sim_host():
    from caffe_mpi_b200 import host_api
    capi.lib()
    r = subprocess.run(["make", "-C", os.path.join(HERE, "sim"), "libtrainsim.so"], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.fail("tests/sim/libtrainsim.so does not build:\n" + r.stdout[-1000:] + r.stderr[-3000:])
    saved = (host_api._lib, host_api._SO, os.environ.get("B2C_NCCL_ARENA"))
    host_api._lib, host_api._SO = None, os.path.join(HERE, "sim", "libtrainsim.so")
    os.environ["B2C_NCCL_ARENA"] = "0"
    try:
        yield host_api
    finally:
        host_api._lib, host_api._SO = saved[0], saved[1]
        if saved[2] is None:
            os.environ.pop("B2C_NCCL_ARENA", None)
        else:
            os.environ["B2C_NCCL_ARENA"] = saved[2]


TWO_DB_NET = ('name: "two_db"\n'
              'layer {{ name: "data" type: "Data" top: "data" data_param {{ source: "{img}" backend: LMDB batch_size: {B} {dp} }} '
              'transform_param {{ scale: 0.0078125 }} }}\n'
              'layer {{ name: "label" type: "Data" top: "label" data_param {{ source: "{lab}" backend: LMDB batch_size: {B} }} }}\n'
              'layer {{ name: "ip" type: "InnerProduct" bottom: "data" top: "ip" inner_product_param {{ num_output: 10 '
              'weight_filler {{ type: "gaussian" std: 0.01 }} }} }}\n'
              'layer {{ name: "loss" type: "SoftmaxWithLoss" bottom: "ip" bottom: "label" top: "loss" }}\n')


def _two_dbs(tmp_path, n):
    rng = np.random.default_rng(n)
    imgs = rng.integers(0, 256, (n, 1, 3, 3), dtype=np.uint8)
    imgs[:, 0, 0, 0] = np.arange(n)
    cls = rng.integers(0, 10, n)
    lmdb_io.write_datum_lmdb(str(tmp_path / "img"), imgs, np.zeros(n, np.int64))
    write_float_lmdb(str(tmp_path / "lab"), cls.astype(np.float32).reshape(n, 1, 1, 1))
    return imgs, cls


@pytest.mark.parametrize("img_parsers", [1, 3])
def test_two_database_layers_in_one_net_stay_aligned(sim_host, tmp_path, monkeypatch, img_parsers):
    """Images (uint8, parser_threads given) and class labels (float datums, automatic parser count) in two Data layers: every step's
    `label` blob is the class of the records in its `data` blob."""
    monkeypatch.delenv("B2C_DATA", raising=False)
    n, B = 31, 4
    imgs, cls = _two_dbs(tmp_path, n)
    t = sim_host.Trainer(TWO_DB_NET.format(img=tmp_path / "img", lab=tmp_path / "lab", B=B, dp="parser_threads: %d" % img_parsers),
                         SOLVER, num_classes=10)
    for i in range(12):
        t.step(1, copy_input=True)
        rec = np.rint(t.get_blob("data").reshape(B, -1)[:, 0] / 0.0078125).astype(int)
        assert list(rec) == [(i * B + j) % n for j in range(B)]
        assert np.array_equal(t.get_blob("label"), cls[rec].astype(np.float32)), f"step {i}"


def test_two_database_layers_need_one_batch_size(sim_host, tmp_path, monkeypatch):
    monkeypatch.delenv("B2C_DATA", raising=False)
    _two_dbs(tmp_path, 8)
    net = TWO_DB_NET.format(img=tmp_path / "img", lab=tmp_path / "lab", B=4, dp="").replace(
        'source: "%s" backend: LMDB batch_size: 4' % (tmp_path / "lab"), 'source: "%s" backend: LMDB batch_size: 2' % (tmp_path / "lab"))
    with pytest.raises(sim_host.HostError, match="must have one batch_size"):
        sim_host.Trainer(net, SOLVER, num_classes=10)


def test_two_solvers_read_aligned_stripes_of_both_databases(sim_host, tmp_path, monkeypatch):
    """Two ranks, the image layer with 3 parser threads and the label layer on the automatic count (1 for float datums): TrainNet gives
    both 3, so each rank's label blob is still the class of the records in its data blob, and the records are the rank's stripe."""
    monkeypatch.delenv("B2C_DATA", raising=False)
    L = sim_host.lib()
    for fn, at in (("sim_use_rank_stream", [C.c_int]), ("fakecuda_set_all_eager", [C.c_int]), ("sim_set_solver_count", [C.c_int])):
        getattr(L, fn).argtypes = at
    L.fakecuda_set_all_eager(0)
    n, B, P, steps = 53, 3, 3, 7
    imgs, cls = _two_dbs(tmp_path, n)
    net = TWO_DB_NET.format(img=tmp_path / "img", lab=tmp_path / "lab", B=B, dp="parser_threads: %d" % P)
    try:
        ranks, uid = [], None
        for r in range(2):
            L.sim_use_rank_stream(r)
            t = sim_host.Trainer(net, SOLVER, num_classes=10, seed=50 + r)
            if r == 0:
                uid = t.new_unique_id()
            t.attach_sync(2, r, uid)
            ranks.append(t)
        for i in range(steps):
            for r, t in enumerate(ranks):                               # both ranks enqueue the step's allreduce before either reads
                L.sim_use_rank_stream(r)
                t.step(1, copy_input=True)
            for r, t in enumerate(ranks):
                L.sim_use_rank_stream(r)
                rec = np.rint(t.get_blob("data").reshape(B, -1)[:, 0] / 0.0078125).astype(int)
                assert list(rec) == [p for p, _ in oracle_batches(n, steps, B, 2, r, P)[i]], f"rank {r} step {i}"
                assert np.array_equal(t.get_blob("label"), cls[rec].astype(np.float32)), f"rank {r} step {i}"
    finally:
        L.sim_use_rank_stream(-1)
        L.sim_set_solver_count(1)


@pytest.mark.parametrize("order", ["database-first", "synthetic-first", "input-layer"])
def test_database_and_synthetic_data_layers_do_not_mix(sim_host, tmp_path, monkeypatch, order):
    """A Data layer whose source does not open falls back to the synthetic source; next to a database layer it would never be
    reloaded, so the net is refused whichever comes first -- and so is an Input layer next to one."""
    monkeypatch.delenv("B2C_DATA", raising=False)
    _two_dbs(tmp_path, 8)
    net = TWO_DB_NET.format(img=tmp_path / "img", lab=tmp_path / "lab", B=4, dp="")
    lab_layer = net[net.index('layer { name: "label"'):net.index('layer { name: "ip"')]
    missing = lab_layer.replace(str(tmp_path / "lab"), str(tmp_path / "no_such_lmdb"))
    if order == "database-first":
        net = net.replace(lab_layer, missing)
    elif order == "synthetic-first":
        img_layer = net[net.index('layer { name: "data"'):net.index('layer { name: "label"')]
        net = net.replace(img_layer + lab_layer, missing + img_layer)
    else:
        net = net.replace(lab_layer, 'layer { name: "label" type: "Input" top: "label" input_param { shape { dim: 4 } } }\n')
    with pytest.raises(sim_host.HostError, match="feeds synthetic data next to Data layers that read databases"):
        sim_host.Trainer(net, SOLVER, num_classes=10)


def test_each_database_layer_draws_its_own_mirror_stream(sim_host, tmp_path, monkeypatch):
    """Two image Data layers over one database, both mirror: true without a random_seed: each draws its own stream, so some item is
    flipped in one layer and not in the other (the first layer keeps the stream a one-layer net draws)."""
    monkeypatch.delenv("B2C_DATA", raising=False)
    imgs, _ = _two_dbs(tmp_path, 16)
    net = TWO_DB_NET.format(img=tmp_path / "img", lab=tmp_path / "lab", B=4, dp="").replace(
        "transform_param { scale: 0.0078125 }", "transform_param { mirror: true }")
    second = net[net.index('layer { name: "data"'):net.index('layer { name: "label"')].replace('"data"', '"data2"')
    two = sim_host.Trainer(net.replace('layer { name: "label"', second + 'layer { name: "label"'), SOLVER, num_classes=10)
    one = sim_host.Trainer(net, SOLVER, num_classes=10)
    differ = False
    for _ in range(4):
        two.step(1, copy_input=True)
        one.step(1, copy_input=True)
        a, b = two.get_blob("data").reshape(4, 3, 3), two.get_blob("data2").reshape(4, 3, 3)
        assert np.array_equal(a, one.get_blob("data").reshape(4, 3, 3))
        for x, y in zip(a, b):
            assert np.array_equal(x, y) or np.array_equal(x, y[:, ::-1])        # the same records, flipped or not
            differ |= not np.array_equal(x, y)
    assert differ

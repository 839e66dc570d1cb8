"""DataLayer's slot protocol without a GPU: the product class (caffe_mpi_b200/host/data_layer.cpp, compiled unchanged) runs on a
stream-order model of the CUDA runtime (tests/sim/fake_cuda.cpp) in which every stream executes either as LATE or as EARLY as the
program's own dependencies -- event waits and host synchronisations -- allow.  Under each combination of extremes for the compute
stream and the copy stream the layer must still deliver, bit for bit, the batches the reference's pipeline would
(CursorManager's records, Fill3Randoms' crops and flips, DataTransformer::Transform's arithmetic): a missing wait between the
parser threads' pinned buffers, the host -> device copies and the transform shows up as a wrong batch.

What this does NOT cover: the transform kernel itself (a host closure stands in for it here; the real one is checked bit-exactly
on hardware by tests/test_layers_extra_gpu.py) and real PCIe / driver behaviour -- tests/test_zz_data_layer_gpu.py is the same
comparison on an H100."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from caffe_mpi_b200 import capi, data_api, lmdb_io
from oracle import layers_oracle as lo
from test_data_cpu import oracle_batches

HERE = os.path.dirname(os.path.abspath(__file__))
NET = ('name: "sim" layer {{ name: "data" type: "Data" top: "data" top: "label" data_param {{ source: "{src}" backend: LMDB batch_size: {B} {dp} }} '
       'transform_param {{ {tp} }} }}')


@pytest.fixture(scope="module")
def sim():
    capi.lib()                                              # libb2c.so must exist (the simulator links it for the host layer's other symbols)
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
    L.sim_batches.argtypes = [C.c_void_p]
    L.sim_batches.restype = C.c_longlong
    L.sim_transform_log.argtypes = [C.POINTER(C.c_ulonglong), C.c_int, C.c_int]
    L.fakecuda_set_eager.argtypes = [C.c_void_p, C.c_int]
    L.fakecuda_set_all_eager.argtypes = [C.c_int]
    L.fakecuda_pending.restype = C.c_ulonglong
    for fn, args in (("cudaMalloc", [C.POINTER(C.c_void_p), C.c_size_t]), ("cudaMallocHost", [C.POINTER(C.c_void_p), C.c_size_t]),
                     ("cudaStreamCreateWithFlags", [C.POINTER(C.c_void_p), C.c_uint]), ("cudaEventCreateWithFlags", [C.POINTER(C.c_void_p), C.c_uint]),
                     ("cudaMemcpyAsync", [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p]), ("cudaStreamSynchronize", [C.c_void_p]),
                     ("cudaEventRecord", [C.c_void_p, C.c_void_p]), ("cudaStreamWaitEvent", [C.c_void_p, C.c_void_p, C.c_uint]),
                     ("cudaEventSynchronize", [C.c_void_p]), ("cudaDeviceSynchronize", [])):
        getattr(L, fn).argtypes = args
    return L


# ---- the simulator itself: it must SEE the hazards it is there to catch ------------------------------------------------------------
def _buf(L, n, host=False):
    p = C.c_void_p()
    assert (L.cudaMallocHost if host else L.cudaMalloc)(C.byref(p), n) == 0
    return p


def _stream(L):
    s = C.c_void_p()
    assert L.cudaStreamCreateWithFlags(C.byref(s), 1) == 0
    return s


def _event(L):
    e = C.c_void_p()
    assert L.cudaEventCreateWithFlags(C.byref(e), 2) == 0
    return e


def test_simulator_reads_a_pinned_source_when_the_copy_runs(sim):
    L = sim
    L.fakecuda_set_all_eager(0)
    src, dst, s = _buf(L, 4, host=True), _buf(L, 4), _stream(L)
    C.memmove(src, b"AAAA", 4)
    L.cudaMemcpyAsync(dst, src, 4, 1, s)
    C.memmove(src, b"BBBB", 4)                               # refilled before the copy was known to have completed
    L.cudaStreamSynchronize(s)
    assert C.string_at(dst, 4) == b"BBBB"                    # the hazard is visible: a lazy copy stream delivers the refill
    C.memmove(src, b"CCCC", 4)
    L.cudaMemcpyAsync(dst, src, 4, 1, s)
    e = _event(L)
    L.cudaEventRecord(e, s)
    L.cudaEventSynchronize(e)                                # the fix: wait for the copy, then refill
    C.memmove(src, b"DDDD", 4)
    L.cudaDeviceSynchronize()
    assert C.string_at(dst, 4) == b"CCCC"


def test_simulator_orders_streams_only_through_events(sim):
    L = sim
    a, b, out = _buf(L, 4), _buf(L, 4), _buf(L, 4, host=True)
    prod, cons = _stream(L), _stream(L)
    C.memmove(a, b"old!", 4)
    new = _buf(L, 4, host=True)
    C.memmove(new, b"new!", 4)
    # consumer forgets to wait for the producer: under a lazy producer it reads the stale buffer
    L.fakecuda_set_all_eager(0)
    L.cudaMemcpyAsync(a, new, 4, 1, prod)
    L.cudaMemcpyAsync(out, a, 4, 2, cons)
    L.cudaStreamSynchronize(cons)
    assert C.string_at(out, 4) == b"old!"
    L.cudaDeviceSynchronize()
    # with the event in place the synchronise on the consumer drags the producer along
    C.memmove(a, b"old!", 4)
    e = _event(L)
    L.cudaMemcpyAsync(a, new, 4, 1, prod)
    L.cudaEventRecord(e, prod)
    L.cudaStreamWaitEvent(cons, e, 0)
    L.cudaMemcpyAsync(out, a, 4, 2, cons)
    L.cudaStreamSynchronize(cons)
    assert C.string_at(out, 4) == b"new!"
    # producer forgets to wait for the previous consumer: under an eager producer the live buffer is overwritten
    C.memmove(a, b"live", 4)
    L.fakecuda_set_eager(prod, 1)
    L.cudaMemcpyAsync(out, a, 4, 2, cons)                    # consumer of "live", still pending (lazy)
    L.cudaMemcpyAsync(a, new, 4, 1, prod)                    # runs at once
    L.cudaStreamSynchronize(cons)
    assert C.string_at(out, 4) == b"new!"                    # the hazard is visible
    # an event wait holds an eager stream back until its dependency has run
    C.memmove(a, b"live", 4)
    L.cudaMemcpyAsync(out, a, 4, 2, cons)
    L.cudaEventRecord(e, cons)
    L.cudaStreamWaitEvent(prod, e, 0)
    L.cudaMemcpyAsync(a, new, 4, 1, prod)
    assert C.string_at(a, 4) == b"live" and L.fakecuda_pending() > 0
    L.cudaStreamSynchronize(prod)
    assert C.string_at(out, 4) == b"live" and C.string_at(a, 4) == b"new!"
    L.fakecuda_set_all_eager(0)


# ---- DataLayer on the simulator -----------------------------------------------------------------------------------------------------
def _db(tmp_path, n, c, h, w):
    rng = np.random.default_rng(200 + n)
    imgs = rng.integers(0, 256, (n, c, h, w), dtype=np.uint8)
    labels = rng.integers(0, 10, n)
    path = str(tmp_path / "lmdb")
    lmdb_io.write_datum_lmdb(path, imgs, labels)
    return path, imgs, labels


MODES = {"all-lazy": (0, 0), "all-eager": (1, 1), "compute-lazy_copy-eager": (0, 1), "compute-eager_copy-lazy": (1, 0)}


@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("P,S,rank", [(1, 1, 0), (2, 1, 0), (3, 2, 1)])
def test_data_layer_delivers_reference_batches_under_extreme_stream_orders(sim, tmp_path, monkeypatch, mode, P, S, rank):
    monkeypatch.delenv("B2C_DATA", raising=False)
    L = sim
    n, Cc, H, W, B, crop, seed, steps = 47, 3, 11, 9, 4, 7, 31, 14
    path, imgs, labels = _db(tmp_path, n, Cc, H, W)
    mean = [104.0, 117.0, 123.0]
    net = NET.format(src=path, B=B, dp="parser_threads: %d" % P,
                     tp="crop_size: %d mirror: true scale: 0.25 random_seed: %d %s" % (crop, seed, " ".join("mean_value: %g" % m for m in mean)))
    L.fakecuda_set_all_eager(0)
    h = L.sim_create(net.encode(), 1701, S, rank)
    assert h, L.sim_last_error().decode()
    compute_eager, copy_eager = MODES[mode]
    L.fakecuda_set_all_eager(copy_eager)                     # every stream but the legacy (compute) one is the layer's copy stream
    L.fakecuda_set_eager(None, compute_eager)
    shp = (C.c_int * 4)()
    L.sim_shape(h, shp)
    assert tuple(shp) == (B, Cc, crop, crop)
    want_batches = oracle_batches(n, steps, B, S, rank, P)
    ho, wo, mir = data_api.transform_draws(seed, True, crop, True, B * steps, H, W)
    got, lab = np.empty((B, Cc, crop, crop), np.float32), np.empty(B, np.float32)
    log = (C.c_ulonglong * 64)()
    L.sim_transform_log(log, 64, 1)
    for i in range(steps):
        assert L.sim_load_batch(h) == 0, L.sim_last_error().decode()
        if i % 7 != 6 and i != steps - 1:
            continue                  # most batches are never read back: several LoadBatch calls in a row meet pending work, and every
                                      # slot is reused while transforms that read it may still be queued (K = P + 1 <= 4 slots)
        assert L.sim_read(h, got.ctypes.data_as(C.c_void_p), lab.ctypes.data_as(C.c_void_p)) == 0, L.sim_last_error().decode()
        pos = [p for p, _ in want_batches[i]]
        want = lo.transform_u8(imgs[pos], (crop, crop), ho[B * i:B * i + B], wo[B * i:B * i + B], mir[B * i:B * i + B], mean, None, 0.25)
        assert np.array_equal(got, want), f"{mode}: batch {i}"
        assert np.array_equal(lab, labels[pos].astype(np.float32)), f"{mode}: labels of batch {i}"
        assert L.sim_batches(h) == i + 1
    # every transform, read back or not, consumed the bytes of ITS batch (a device slot overwritten early shows up here)
    assert L.sim_transform_log(log, 64, 1) == steps
    assert [int(log[i]) for i in range(steps)] == [int(imgs[[p for p, _ in want_batches[i]]].astype(np.uint64).sum()) for i in range(steps)]
    L.sim_destroy(h)
    L.fakecuda_set_all_eager(0)


def test_data_layer_mean_file_and_no_crop_on_the_simulator(sim, tmp_path, monkeypatch):
    monkeypatch.delenv("B2C_DATA", raising=False)
    L = sim
    path, imgs, labels = _db(tmp_path, 10, 1, 6, 5)
    mean = np.random.default_rng(1).uniform(90, 130, (1, 1, 6, 5)).astype(np.float32)
    mp = str(tmp_path / "mean.binaryproto")
    data_api.blobproto_save(mp, mean)
    h = L.sim_create(NET.format(src=path, B=4, dp="", tp='mean_file: "%s" scale: 0.00390625' % mp).encode(), 1, 1, 0)
    assert h, L.sim_last_error().decode()
    got, lab = np.empty((4, 1, 6, 5), np.float32), np.empty(4, np.float32)
    want_batches = oracle_batches(10, 4, 4, 1, 0, 1)
    zeros = np.zeros(4, np.int32)
    for i in range(4):                                       # batch 2 wraps: records 8, 9, 0, 1
        assert L.sim_load_batch(h) == 0 and L.sim_read(h, got.ctypes.data_as(C.c_void_p), lab.ctypes.data_as(C.c_void_p)) == 0
        pos = [p for p, _ in want_batches[i]]
        assert np.array_equal(got, lo.transform_u8(imgs[pos], (6, 5), zeros, zeros, zeros, None, mean[0], 0.00390625))
        assert np.array_equal(lab, labels[pos].astype(np.float32))
    L.sim_destroy(h)
    # what the layer refuses at set-up (data_transformer.cpp:21-22, :198-200)
    bad = L.sim_create(NET.format(src=path, B=4, dp="", tp='mean_file: "%s" mean_value: 1' % mp).encode(), 1, 1, 0)
    assert not bad and "Cannot specify mean_file and mean_value at the same time" in L.sim_last_error().decode()
    data_api.blobproto_save(mp, np.zeros((1, 1, 5, 5), np.float32))
    bad = L.sim_create(NET.format(src=path, B=4, dp="", tp='mean_file: "%s"' % mp).encode(), 1, 1, 0)
    assert not bad and "does not have the datums'" in L.sim_last_error().decode()


# ---- the reference's own DataLayer tests (src/caffe/test/test_data_layer.cpp), on the simulator ------------------------------------------
def _fill(tmp_path, unique_pixels):
    """DataLayerTest::Fill (test_data_layer.cpp:44-70): five 2x3x4 datums under the keys "0".."4", label = index; either every pixel
    of an image is unique and all images equal, or every image is one constant."""
    items = []
    for i in range(5):
        data = np.array([j if unique_pixels else i for j in range(24)], np.uint8).reshape(2, 3, 4)
        items.append((str(i).encode(), lmdb_io.datum_bytes(data, i)))
    path = str(tmp_path / ("db%d" % unique_pixels))
    lmdb_io.write_lmdb(path, items)
    return path


def _layer(L, path, tp, seed=1701):
    h = L.sim_create(NET.format(src=path, B=5, dp="parser_threads: 3", tp=tp).encode(), seed, 1, 0)
    assert h, L.sim_last_error().decode()
    shp = (C.c_int * 4)()
    L.sim_shape(h, shp)
    return h, tuple(shp)


def _forward(L, h, shape):
    data, label = np.empty(shape, np.float32), np.empty(shape[0], np.float32)
    assert L.sim_load_batch(h) == 0 and L.sim_read(h, data.ctypes.data_as(C.c_void_p), label.ctypes.data_as(C.c_void_p)) == 0
    return data, label


def test_reference_TestReadLMDB(sim, tmp_path, monkeypatch):
    monkeypatch.delenv("B2C_DATA", raising=False)
    L = sim
    h, shape = _layer(L, _fill(tmp_path, False), "scale: 3")
    assert shape == (5, 2, 3, 4)
    for _ in range(100):                                      # test_data_layer.cpp:98-109
        data, label = _forward(L, h, shape)
        assert label.tolist() == [0, 1, 2, 3, 4]
        assert np.array_equal(data, np.broadcast_to((3.0 * np.arange(5, dtype=np.float32)).reshape(5, 1, 1, 1), shape))
    L.sim_destroy(h)


def test_reference_TestReadCropTrainLMDB(sim, tmp_path, monkeypatch):
    monkeypatch.delenv("B2C_DATA", raising=False)
    L = sim
    h, shape = _layer(L, _fill(tmp_path, True), "scale: 3 crop_size: 1")
    assert shape == (5, 2, 1, 1)
    for _ in range(2):                                        # test_data_layer.cpp:204-227, TRAIN branch
        data, label = _forward(L, h, shape)
        assert label.tolist() == [0, 1, 2, 3, 4]
        centre = np.array([3.0 * 5, 3.0 * 17], np.float32)
        assert int((data.reshape(5, 2) == centre).sum()) < 10   # not the centre crop all ten times
        # every value is 3 x a pixel of its own channel (channel 0 holds 0..11, channel 1 holds 12..23)
        px = data.reshape(5, 2) / 3
        assert ((px[:, 0] >= 0) & (px[:, 0] < 12) & (px[:, 1] >= 12) & (px[:, 1] < 24)).all()
    L.sim_destroy(h)


def _crop_sequence(L, path, seed, tp="crop_size: 1 mirror: true"):
    h, shape = _layer(L, path, tp, seed=seed)
    seq = []
    for _ in range(2):
        data, label = _forward(L, h, shape)
        assert label.tolist() == [0, 1, 2, 3, 4]
        seq.append(data.reshape(-1).copy())
    L.sim_destroy(h)
    return np.concatenate(seq)


def test_reference_TestReadCropTrainSequenceSeeded_and_Unseeded(sim, tmp_path, monkeypatch):
    monkeypatch.delenv("B2C_DATA", raising=False)
    L = sim
    path = _fill(tmp_path, True)
    first = _crop_sequence(L, path, 1701)
    assert np.array_equal(_crop_sequence(L, path, 1701), first)          # same seed, same crops and flips (:256-286)
    other = _crop_sequence(L, path, 1702)                                # a solver that went on drawing: another stream (:328-352)
    assert int((other == first).sum()) < 20
    # transform_param.random_seed pins the stream whatever the solver's seed is (data_transformer.cpp:733-736)
    a = _crop_sequence(L, path, 1, tp="crop_size: 1 mirror: true random_seed: 9")
    b = _crop_sequence(L, path, 2, tp="crop_size: 1 mirror: true random_seed: 9")
    assert np.array_equal(a, b)


# ---- encoded datums of DIFFERENT sizes: the parser threads decode and cut the crop window ---------------------------------------------------------
@pytest.mark.parametrize("P", [1, 3])
def test_encoded_datums_of_varying_size_are_cropped_by_the_parser_threads(sim, tmp_path, monkeypatch, P):
    """A database of original image files (convert_imageset --encoded without a resize): every datum has its own height and width,
    which the reference allows as long as crop_size is set (data_layer.cpp:262-271, "crop might help here").  The parser threads decode
    each file and cut the window DataTransformer::Transform would (h_off = rand1 % (H - crop + 1), data_transformer.cpp:219-226) from
    the Fill3Randoms draws the layer makes in batch order; the device only flips.  Expected values: cv2.imdecode + those rules."""
    cv2 = pytest.importorskip("cv2")
    from test_data_cpu import _mt19937
    monkeypatch.delenv("B2C_DATA", raising=False)
    L = sim
    rng = np.random.default_rng(8)
    n, B, crop, seed, steps = 11, 3, 12, 99, 6
    files, labels = [], rng.integers(0, 10, n)
    for i in range(n):
        h, w = int(rng.integers(crop, 40)), int(rng.integers(crop, 40))
        img = cv2.resize(rng.integers(0, 256, (5, 5, 3), dtype=np.uint8), (w, h), interpolation=cv2.INTER_CUBIC)
        ok, enc = cv2.imencode(".jpg" if i % 3 else ".png", img, [cv2.IMWRITE_JPEG_QUALITY, 85] if i % 3 else [])
        files.append(enc.tobytes())
    path = str(tmp_path / "orig_db")
    env = data_api.LMDB(path, "NEW")
    for i, f in enumerate(files):
        env.put(lmdb_io.caffe_key(i, "im%d" % i), data_api.datum_serialize(0, 0, 0, f, int(labels[i]), encoded=True))
    env.commit()
    env.close()
    decoded = [cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_UNCHANGED).transpose(2, 0, 1) for f in files]
    L.fakecuda_set_all_eager(0)
    h = L.sim_create(NET.format(src=path, B=B, dp="parser_threads: %d" % P, tp="crop_size: %d mirror: true scale: 0.5 mean_value: 100 random_seed: %d" % (crop, seed)).encode(),
                     7, 1, 0)
    assert h, L.sim_last_error().decode()
    shp = (C.c_int * 4)()
    L.sim_shape(h, shp)
    assert tuple(shp) == (B, 3, crop, crop)
    raw = _mt19937(seed, 3 * B * (steps + P + 2)).tolist()                     # three draws per item, batch after batch
    want_batches = oracle_batches(n, steps, B, 1, 0, P)
    got, lab = np.empty((B, 3, crop, crop), np.float32), np.empty(B, np.float32)
    for i in range(steps):
        assert L.sim_load_batch(h) == 0, L.sim_last_error().decode()
        assert L.sim_read(h, got.ctypes.data_as(C.c_void_p), lab.ctypes.data_as(C.c_void_p)) == 0
        for j, (pos, _) in enumerate(want_batches[i]):
            r0, r1, r2 = ((raw[3 * (B * i + j) + k] + 1) & 0xFFFFFFFF for k in range(3))
            img = decoded[pos]
            ho, wo = r1 % (img.shape[1] - crop + 1), r2 % (img.shape[2] - crop + 1)
            win = (img[:, ho:ho + crop, wo:wo + crop].astype(np.float32) - np.float32(100.0)) * np.float32(0.5)
            if r0 % 2:
                win = win[:, :, ::-1]
            assert np.array_equal(got[j], win), (i, j, pos)
            assert lab[j] == labels[pos]
    L.sim_destroy(h)

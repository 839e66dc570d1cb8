"""ctypes binding of host/b2h_data_capi.cpp: the input pipeline's host half (db::LMDB cursor, Datum, DataReader, the
DataTransformer's draws).  Nothing here touches the device."""
import ctypes as C

import numpy as np

from . import host_api

_ready = False


class DataError(RuntimeError):
    pass


def lib():
    global _ready
    L = host_api.lib()
    if not _ready:
        vp, i, ll = C.c_void_p, C.c_int, C.c_longlong
        L.b2h_data_last_error.restype = C.c_char_p
        L.b2h_lmdb_exists.argtypes = [C.c_char_p]
        L.b2h_lmdb_open.restype = vp
        L.b2h_lmdb_open.argtypes = [C.c_char_p]
        L.b2h_lmdb_open_mode.restype = vp
        L.b2h_lmdb_open_mode.argtypes = [C.c_char_p, i]
        L.b2h_lmdb_put.argtypes = [vp, C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t]
        L.b2h_lmdb_commit.argtypes = [vp]
        L.b2h_lmdb_close.argtypes = [vp]
        L.b2h_lmdb_stat.argtypes = [vp, C.POINTER(ll), C.POINTER(C.c_uint), C.POINTER(C.c_uint), C.POINTER(C.c_ulonglong)]
        for fn in ("b2h_lmdb_seek_to_first", "b2h_lmdb_next", "b2h_lmdb_valid"):
            getattr(L, fn).argtypes = [vp]
        L.b2h_lmdb_current.argtypes = [vp, C.POINTER(vp), C.POINTER(C.c_size_t), C.POINTER(vp), C.POINTER(C.c_size_t)]
        L.b2h_datum_parse.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(ll), C.POINTER(vp), C.POINTER(C.c_size_t), C.POINTER(C.c_float), i,
                                      C.POINTER(i)]
        L.b2h_datum_serialize.restype = ll
        L.b2h_datum_serialize.argtypes = [i, i, i, C.c_char_p, C.c_size_t, i, i, C.POINTER(C.c_float), i, C.c_char_p, C.c_size_t]
        L.b2h_blobproto_load.argtypes = [C.c_char_p, C.POINTER(i), C.POINTER(i), C.POINTER(ll), vp]
        L.b2h_blobproto_save.argtypes = [C.c_char_p, i, C.POINTER(i), C.POINTER(C.c_float), i]
        L.b2h_jpeg_decode.argtypes = [C.c_char_p, C.c_size_t, i, C.POINTER(i), vp, C.c_size_t]
        L.b2h_data_reader_create.restype = vp
        L.b2h_data_reader_create.argtypes = [C.c_char_p, i, i, i, i, i, i, i, i]
        L.b2h_data_reader_destroy.argtypes = [vp]
        L.b2h_data_reader_info.argtypes = [vp, C.POINTER(i), C.POINTER(ll), C.POINTER(ll)]
        L.b2h_data_reader_first_record.restype = ll
        L.b2h_data_reader_first_record.argtypes = [vp, ll]
        L.b2h_data_reader_next.argtypes = [vp, vp, vp, vp, C.POINTER(ll)]
        L.b2h_transform_draws.argtypes = [C.c_ulonglong, i, i, i, i, i, i, vp, vp, vp]
        _ready = True
    return L


def _err():
    return DataError(lib().b2h_data_last_error().decode())


def lmdb_exists(source):
    return bool(lib().b2h_lmdb_exists(source.encode()))


class LMDB:
    """caffe::db::LMDB (mode "READ", "WRITE" or "NEW") plus one LMDBCursor and one pending LMDBTransaction on it."""

    def __init__(self, source, mode="READ"):
        self._h = lib().b2h_lmdb_open_mode(source.encode(), {"READ": 0, "WRITE": 1, "NEW": 2}[mode])
        if not self._h:
            raise _err()

    def put(self, key, value):
        if lib().b2h_lmdb_put(self._h, key, len(key), value, len(value)) != 0:
            raise _err()

    def commit(self):
        if lib().b2h_lmdb_commit(self._h) != 0:
            raise _err()

    def stat(self):
        n, ps, d, t = C.c_longlong(), C.c_uint(), C.c_uint(), C.c_ulonglong()
        if lib().b2h_lmdb_stat(self._h, C.byref(n), C.byref(ps), C.byref(d), C.byref(t)) != 0:
            raise _err()
        return dict(entries=n.value, page_size=ps.value, depth=d.value, txnid=t.value)

    def seek_to_first(self):
        r = lib().b2h_lmdb_seek_to_first(self._h)
        if r < 0:
            raise _err()
        return bool(r)

    def next(self):
        r = lib().b2h_lmdb_next(self._h)
        if r < 0:
            raise _err()
        return bool(r)

    def valid(self):
        return bool(lib().b2h_lmdb_valid(self._h))

    def current(self):
        k, v, kn, vn = C.c_void_p(), C.c_void_p(), C.c_size_t(), C.c_size_t()
        if lib().b2h_lmdb_current(self._h, C.byref(k), C.byref(kn), C.byref(v), C.byref(vn)) != 0:
            raise _err()
        return C.string_at(k.value, kn.value), C.string_at(v.value, vn.value)

    def items(self):
        """Every (key, value) from the first record on: SeekToFirst, then Next until the cursor turns invalid."""
        out = []
        ok = self.seek_to_first()
        while ok:
            out.append(self.current())
            ok = self.next()
        return out

    def close(self):
        if self._h:
            lib().b2h_lmdb_close(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def datum_parse(buf):
    """dict of the Datum's fields, or None if the bytes do not parse (Datum::ParseFromArray returning false)."""
    out = (C.c_longlong * 6)()
    data, size, nf = C.c_void_p(), C.c_size_t(), C.c_int()
    cap = max(1, len(buf) // 4)
    fl = (C.c_float * cap)()
    if not lib().b2h_datum_parse(buf, len(buf), out, C.byref(data), C.byref(size), fl, cap, C.byref(nf)):
        return None
    return dict(channels=out[0], height=out[1], width=out[2], label=out[3], encoded=bool(out[4]), record_id=out[5],
                data=C.string_at(data.value, size.value) if size.value else b"", float_data=[fl[k] for k in range(min(nf.value, cap))])


def datum_serialize(channels, height, width, data, label, encoded=False, float_data=None):
    fd = list(float_data or [])
    cap = len(data) + 4 * len(fd) + 5 * len(fd) + 64
    out = C.create_string_buffer(cap)
    n = lib().b2h_datum_serialize(channels, height, width, data, len(data), label, int(encoded), (C.c_float * max(1, len(fd)))(*fd), len(fd),
                                  out, cap)
    if n < 0:
        raise _err()
    return out.raw[:n]


def jpeg_decode(buf, force_color=False):
    """uint8 [C][H][W] (channels B, G, R like cv2) of a baseline JPEG file's bytes; DataError for what the decoder does not take."""
    chw = (C.c_int * 3)()
    if lib().b2h_jpeg_decode(buf, len(buf), int(force_color), chw, None, 0) != 0:
        raise _err()
    out = np.empty((chw[0], chw[1], chw[2]), np.uint8)
    if lib().b2h_jpeg_decode(buf, len(buf), int(force_color), chw, out.ctypes.data_as(C.c_void_p), out.size) != 0:
        raise _err()
    return out


def blobproto_load(path):
    nd, shp, cnt = C.c_int(), (C.c_int * 8)(), C.c_longlong()
    if lib().b2h_blobproto_load(path.encode(), C.byref(nd), shp, C.byref(cnt), None) != 0:
        raise _err()
    arr = np.empty(cnt.value, np.float32)
    if lib().b2h_blobproto_load(path.encode(), C.byref(nd), shp, C.byref(cnt), arr.ctypes.data_as(C.c_void_p)) != 0:
        raise _err()
    return arr.reshape([shp[k] for k in range(nd.value)])


def blobproto_save(path, arr, raw=False):
    arr = np.ascontiguousarray(arr, np.float32)
    if lib().b2h_blobproto_save(path.encode(), arr.ndim, (C.c_int * arr.ndim)(*arr.shape), arr.ctypes.data_as(C.POINTER(C.c_float)), int(raw)) != 0:
        raise _err()


class DataReader:
    """caffe::DataReader: parser threads over an LMDB with the reference's (node, solver, thread) record partition."""

    def __init__(self, source, batch_size, solver_count=1, solver_rank=0, node_count=1, node_rank=0, parser_threads=1, depth=2,
                 force_encoded_color=False):
        self._h = lib().b2h_data_reader_create(source.encode(), batch_size, solver_count, solver_rank, node_count, node_rank, parser_threads, depth,
                                               int(force_encoded_color))
        if not self._h:
            raise _err()
        chw, n, fc = (C.c_int * 3)(), C.c_longlong(), C.c_longlong()
        lib().b2h_data_reader_info(self._h, chw, C.byref(n), C.byref(fc))
        self.shape = (chw[0], chw[1], chw[2])
        self.entries, self.full_cycle, self.batch_size = n.value, fc.value, batch_size
        db = LMDB(source)                                # the batches are floats when the first datum carries float_data only
        first = datum_parse(db.current()[1])
        db.close()
        self.dtype = np.float32 if first["float_data"] and not first["data"] else np.uint8

    def first_record(self, batch):
        return lib().b2h_data_reader_first_record(self._h, batch)

    def next(self):
        """(data [B][C][H][W] of self.dtype, label float32 [B], record_id uint32 [B], batch_id)"""
        data = np.empty((self.batch_size,) + self.shape, self.dtype)
        label = np.empty(self.batch_size, np.float32)
        ids = np.empty(self.batch_size, np.uint32)
        bid = C.c_longlong()
        if lib().b2h_data_reader_next(self._h, data.ctypes.data_as(C.c_void_p), label.ctypes.data_as(C.c_void_p), ids.ctypes.data_as(C.c_void_p),
                                      C.byref(bid)) != 0:
            raise _err()
        return data, label, ids, bid.value

    def close(self):
        if self._h:
            lib().b2h_data_reader_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def transform_draws(seed, mirror, crop, train, n, datum_h, datum_w):
    """(h_off int32 [n], w_off int32 [n], do_mirror uint8 [n]) of n consecutive datums (DataTransformer::Fill3Randoms + Transform)."""
    h, w, m = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.uint8)
    if lib().b2h_transform_draws(seed, int(mirror), crop, int(train), n, datum_h, datum_w, h.ctypes.data_as(C.c_void_p),
                                 w.ctypes.data_as(C.c_void_p), m.ctypes.data_as(C.c_void_p)) != 0:
        raise _err()
    return h, w, m

"""ctypes binding of the flat C test/driver API (host/b2h_capi.cpp) over the C++ host layer libb2caffe.so."""
import ctypes as C
import os

import numpy as np

from . import capi

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libb2caffe.so")
_lib = None
_f32 = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")


class HostError(RuntimeError):
    pass


def lib():
    global _lib
    if _lib is None:
        capi.lib()   # libb2c.so first (RTLD_GLOBAL)
        if not os.path.exists(_SO):
            raise HostError(f"{_SO} missing: run __graft_entry__.build()")
        L = C.CDLL(_SO)
        i, vp, f, ip = C.c_int, C.c_void_p, C.c_float, C.POINTER(C.c_int)
        szp = C.POINTER(C.c_size_t)
        L.b2h_last_error.restype = C.c_char_p
        L.b2h_registry_has.argtypes = [C.c_char_p]
        L.b2h_conv_create.restype = vp
        L.b2h_conv_create.argtypes = [i, i, i, ip, i, ip, i, ip, i, ip, i, i, i, i]
        L.b2h_conv_setup.argtypes = [vp, i, ip]
        L.b2h_conv_top_shape.argtypes = [vp, ip, ip]
        L.b2h_conv_num_blobs.argtypes = [vp]
        L.b2h_conv_blob_count.argtypes = [vp, i]
        L.b2h_conv_blob_count.restype = C.c_longlong
        L.b2h_conv_set_blob.argtypes = [vp, i, i, _f32]
        L.b2h_conv_get_blob.argtypes = [vp, i, i, _f32]
        L.b2h_conv_forward.argtypes = [vp, _f32, _f32]
        L.b2h_conv_backward.argtypes = [vp, _f32, vp, i]
        L.b2h_conv_algo_used.argtypes = [vp, i]
        L.b2h_conv_destroy.argtypes = [vp]
        L.b2h_solver_create.restype = vp
        L.b2h_solver_create.argtypes = [f, C.c_char_p, f, f, i, i, f, f, C.c_char_p, i, i, i, ip, i, f, f]
        L.b2h_solver_create_typed.restype = vp
        L.b2h_solver_create_typed.argtypes = [C.c_char_p, f, C.c_char_p, f, f, i, i, f, f, C.c_char_p, i, i, i, ip, i, f, f, f, f, f]
        L.b2h_solver_destroy.argtypes = [vp]
        L.b2h_solver_lr_at.argtypes = [vp, i]
        L.b2h_solver_lr_at.restype = f
        L.b2h_solver_momentum_at.argtypes = [vp, i]
        L.b2h_solver_momentum_at.restype = f
        L.b2h_plan_buckets.argtypes = [i, szp, i, i, ip, ip, szp, szp]
        L.b2h_divide_batch_size.argtypes = [i, i]
        L.b2h_solver_set_params.argtypes = [vp, i, szp, C.POINTER(f), C.POINTER(f)]
        L.b2h_solver_set.argtypes = [vp, i, i, _f32]
        L.b2h_solver_get.argtypes = [vp, i, i, _f32]
        L.b2h_solver_attach_sync.argtypes = [vp, i, i, C.c_char_p, i]
        L.b2h_solver_step.argtypes = [vp]
        L.b2h_solver_iter.argtypes = [vp]
        L.b2h_solver_set_clip_gradients.argtypes = [vp, f]
        L.b2h_solver_clip_state.argtypes = [vp, C.POINTER(f), C.POINTER(f), C.POINTER(C.c_longlong)]
        L.b2h_trainer_clip_state.argtypes = [vp, C.POINTER(f), C.POINTER(f), C.POINTER(C.c_longlong)]
        L.b2h_clip_slots.argtypes = [i, szp, szp]
        L.b2h_clip_slots.restype = C.c_longlong
        _lib = L
    return _lib


def _ck(rc):
    if rc != 0:
        raise HostError(lib().b2h_last_error().decode())


def _ia(v):
    return (C.c_int * len(v))(*[int(a) for a in v])


class ConvolutionLayer:
    """caffe::ConvolutionLayer created through LayerRegistry::CreateLayer({type: "Convolution"})."""

    def __init__(self, num_output, kernel, stride=(), pad=(), dilation=(), group=1, bias_term=True,
                 engine=capi.ENGINE_DEFAULT, math=capi.MATH_FP32, force_nd=False):
        as_list = lambda v: [v] if isinstance(v, int) else list(v)
        k, s, p, d = as_list(kernel), as_list(stride), as_list(pad), as_list(dilation)
        self._h = lib().b2h_conv_create(num_output, int(bias_term), len(k), _ia(k), len(s), _ia(s), len(p), _ia(p), len(d), _ia(d),
                                        group, engine, math, int(force_nd))
        if not self._h:
            raise HostError(lib().b2h_last_error().decode())

    def setup(self, bottom_shape):
        _ck(lib().b2h_conv_setup(self._h, len(bottom_shape), _ia(bottom_shape)))
        self.bottom_shape = tuple(bottom_shape)
        n, shp = C.c_int(), (C.c_int * 16)()
        lib().b2h_conv_top_shape(self._h, C.byref(n), shp)
        self.top_shape = tuple(shp[i] for i in range(n.value))
        return self.top_shape

    def num_blobs(self):
        return lib().b2h_conv_num_blobs(self._h)

    def set_blob(self, i, arr, diff=False):
        _ck(lib().b2h_conv_set_blob(self._h, i, int(diff), np.ascontiguousarray(arr, np.float32).reshape(-1)))

    def get_blob(self, i, diff=False):
        out = np.empty(lib().b2h_conv_blob_count(self._h, i), np.float32)
        _ck(lib().b2h_conv_get_blob(self._h, i, int(diff), out))
        return out

    def forward(self, x):
        y = np.empty(self.top_shape, np.float32)
        _ck(lib().b2h_conv_forward(self._h, np.ascontiguousarray(x, np.float32).reshape(-1), y.reshape(-1)))
        return y

    def backward(self, dy, propagate_down=True):
        dx = np.empty(self.bottom_shape, np.float32) if propagate_down else None
        _ck(lib().b2h_conv_backward(self._h, np.ascontiguousarray(dy, np.float32).reshape(-1),
                                    dx.ctypes.data_as(C.c_void_p) if dx is not None else None, int(propagate_down)))
        return dx

    def algo_used(self, op):
        return lib().b2h_conv_algo_used(self._h, op)

    def __del__(self):
        if getattr(self, "_h", None) and _lib is not None:
            _lib.b2h_conv_destroy(self._h)
            self._h = None


class SGDSolver:
    """caffe::SGDSolver over a standalone arena.  `type` picks the update (SGD, Nesterov, AdaGrad, RMSProp, AdaDelta, Adam);
    delta, momentum2 and rms_decay are the SolverParameter fields those read.  get(i, 3) is the second history (AdaDelta, Adam).
    clip_gradients >= 0 scales every step's gradient to that global L2 norm when it is larger (negative: off)."""

    def __init__(self, base_lr=0.01, lr_policy="fixed", gamma=0.1, power=1.0, stepsize=1, max_iter=1, momentum=0.0,
                 weight_decay=0.0, regularization_type="L2", iter_size=1, reduce_buckets=6, stepvalue=(), rampup_interval=0,
                 rampup_lr=0.0, min_lr=0.0, type="SGD", delta=1e-8, momentum2=0.999, rms_decay=0.0, clip_gradients=-1.0):
        sv = list(stepvalue)
        self._h = lib().b2h_solver_create_typed(type.encode(), base_lr, lr_policy.encode(), gamma, power, stepsize, max_iter, momentum,
                                                weight_decay, regularization_type.encode(), iter_size, reduce_buckets, len(sv),
                                                _ia(sv) if sv else None, rampup_interval, rampup_lr, min_lr, delta, momentum2, rms_decay)
        if not self._h:
            raise HostError(lib().b2h_last_error().decode())
        if clip_gradients != -1.0:
            _ck(lib().b2h_solver_set_clip_gradients(self._h, clip_gradients))

    def clip_state(self):
        """(norm, factor, clipped_count): the last step's gradient norm and scale factor, and the steps clipped so far."""
        return _clip_state(lib().b2h_solver_clip_state, self._h)

    def lr_at(self, it):
        v = lib().b2h_solver_lr_at(self._h, it)
        if v < 0:
            raise HostError(lib().b2h_last_error().decode())
        return float(v)

    def momentum_at(self, it):
        """SGDSolver::GetMomentum at iteration `it` (momentum_policy fixed, poly or opt)"""
        v = lib().b2h_solver_momentum_at(self._h, it)
        if v != v:
            raise HostError(lib().b2h_last_error().decode())
        return float(v)

    def set_params(self, counts, lr_mult=None, decay_mult=None):
        n = len(counts)
        lr = lr_mult or [1.0] * n
        dc = decay_mult or [1.0] * n
        _ck(lib().b2h_solver_set_params(self._h, n, (C.c_size_t * n)(*counts), (C.c_float * n)(*lr), (C.c_float * n)(*dc)))
        self.counts = list(counts)

    def set(self, i, arr, diff=False):
        _ck(lib().b2h_solver_set(self._h, i, int(diff), np.ascontiguousarray(arr, np.float32).reshape(-1)))

    def get(self, i, what=0):
        out = np.empty(self.counts[i], np.float32)
        _ck(lib().b2h_solver_get(self._h, i, what, out))
        return out

    def new_unique_id(self):
        buf = C.create_string_buffer(128)
        _ck(lib().b2h_solver_attach_sync(self._h, 1, 0, buf, 1))
        return buf.raw

    def attach_sync(self, nranks, rank, id_bytes):
        buf = C.create_string_buffer(bytes(id_bytes), 128)
        _ck(lib().b2h_solver_attach_sync(self._h, nranks, rank, buf, 0))

    def step(self):
        _ck(lib().b2h_solver_step(self._h))

    def iter(self):
        return lib().b2h_solver_iter(self._h)

    def __del__(self):
        if getattr(self, "_h", None) and _lib is not None:
            _lib.b2h_solver_destroy(self._h)
            self._h = None


def _clip_state(fn, h):
    n, f = C.c_float(), C.c_float()
    c = C.c_longlong()
    _ck(fn(h, C.byref(n), C.byref(f), C.byref(c)))
    return n.value, f.value, c.value


def clip_slots(counts):
    """(first norm partial of each param, partial count) for params with these element counts, in arena order"""
    n = len(counts)
    out = (C.c_size_t * max(1, n))()
    total = lib().b2h_clip_slots(n, (C.c_size_t * max(1, n))(*counts), out)
    return [out[i] for i in range(n)], int(total)


def plan_buckets(counts, reduce_buckets=6):
    n = len(counts)
    mx = n + 1
    f, t = (C.c_int * mx)(), (C.c_int * mx)()
    off, cnt = (C.c_size_t * mx)(), (C.c_size_t * mx)()
    nb = lib().b2h_plan_buckets(n, (C.c_size_t * n)(*counts), reduce_buckets, mx, f, t, off, cnt)
    if nb < 0:
        raise HostError(lib().b2h_last_error().decode())
    return [(f[i], t[i], off[i], cnt[i]) for i in range(nb)]


def divide_batch_size(total, solver_count):
    return lib().b2h_divide_batch_size(total, solver_count)


# ---------------------------------------------------------------------------------------------- prototxt / Net
class Net:
    """caffe::Net graph built from a prototxt (file path, or text with is_text=True) by the C++ host layer."""

    def __init__(self, path_or_text, phase="TRAIN", batch_override=0, is_text=False, default_channels=3, default_size=224):
        L = lib()
        L.b2h_net_create.restype = C.c_void_p
        L.b2h_net_create.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
        self._h = L.b2h_net_create(path_or_text.encode(), int(is_text), 1 if phase == "TEST" else 0, batch_override,
                                   default_channels, default_size)
        if not self._h:
            raise HostError(L.b2h_last_error().decode())
        for fn in ("b2h_net_num_layers", "b2h_net_num_convs", "b2h_net_num_params", "b2h_net_reduce_buckets", "b2h_net_destroy"):
            getattr(L, fn).argtypes = [C.c_void_p]

    def layers(self):
        L = lib()
        L.b2h_net_layer.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_char_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
        out = []
        for i in range(L.b2h_net_num_layers(self._h)):
            nm, ty = C.create_string_buffer(256), C.create_string_buffer(256)
            na, shp = C.c_int(), (C.c_int * 8)()
            L.b2h_net_layer(self._h, i, nm, ty, 256, C.byref(na), shp)
            out.append((nm.value.decode(), ty.value.decode(), tuple(shp[k] for k in range(na.value))))
        return out

    def top_shape(self, layer, top):
        """The shape Net inferred for top `top` of layer `layer`."""
        L = lib()
        L.b2h_net_top_shape.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
        na, shp = C.c_int(), (C.c_int * 8)()
        _ck(L.b2h_net_top_shape(self._h, layer, top, C.byref(na), shp))
        return tuple(shp[k] for k in range(na.value))

    def loss_params(self, layer):
        """The class-axis parameters of a layer: softmax_param.axis, loss_param (ignore_label or None, normalization name) and
        accuracy_param (axis, top_k, ignore_label or None), axes canonical."""
        L = lib()
        L.b2h_net_loss_params.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int), C.c_int]
        o = (C.c_int * 8)()
        _ck(L.b2h_net_loss_params(self._h, layer, o, 8))
        return {"softmax_axis": o[0], "ignore_label": o[2] if o[1] else None, "normalization": capi.LOSS_NORMS[o[3]],
                "accuracy_axis": o[4], "top_k": o[5], "accuracy_ignore_label": o[7] if o[6] else None}

    def conv_layers(self):
        L = lib()
        L.b2h_net_conv.argtypes = [C.c_void_p, C.c_int, C.POINTER(capi.ConvParams), C.POINTER(C.c_int), C.c_char_p, C.c_int]
        out = []
        for i in range(L.b2h_net_num_convs(self._h)):
            p, pd, nm = capi.ConvParams(), C.c_int(), C.create_string_buffer(256)
            L.b2h_net_conv(self._h, i, C.byref(p), C.byref(pd), nm, 256)
            out.append((nm.value.decode(), p, bool(pd.value)))
        return out

    def learnable_params(self):
        L = lib()
        L.b2h_net_param.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_size_t), C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_char_p, C.c_int]
        out = []
        for i in range(L.b2h_net_num_params(self._h)):
            cnt, lr, dc, nm = C.c_size_t(), C.c_float(), C.c_float(), C.create_string_buffer(256)
            L.b2h_net_param(self._h, i, C.byref(cnt), C.byref(lr), C.byref(dc), nm, 256)
            out.append((nm.value.decode(), cnt.value, lr.value, dc.value))
        return out

    def net_params(self):
        """Every layer's parameter blobs, sharers included: [(layer, param name, owner, learnable id)].  owner is the index of the
        owning blob in this list (-1: the blob owns its storage); learnable id indexes learnable_params()."""
        L = lib()
        L.b2h_net_net_param.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_char_p, C.c_char_p, C.c_int]
        L.b2h_net_num_net_params.argtypes = [C.c_void_p]
        out = []
        for i in range(L.b2h_net_num_net_params(self._h)):
            ow, lid, nm, pn = C.c_int(), C.c_int(), C.create_string_buffer(256), C.create_string_buffer(256)
            L.b2h_net_net_param(self._h, i, C.byref(ow), C.byref(lid), nm, pn, 256)
            out.append((nm.value.decode(), pn.value.decode(), ow.value, lid.value))
        return out

    def reduce_buckets(self):
        return lib().b2h_net_reduce_buckets(self._h)

    def backward_plan(self):
        """Per layer (loss pruning included): (runs backward, [gradient to bottom b for each bottom])."""
        L = lib()
        L.b2h_net_layer_backward.restype = C.c_longlong
        L.b2h_net_layer_backward.argtypes = [C.c_void_p, C.c_int]
        L.b2h_net_layer_bottoms.argtypes = [C.c_void_p, C.c_int]
        out = []
        for i in range(L.b2h_net_num_layers(self._h)):
            v = L.b2h_net_layer_backward(self._h, i)
            out.append((bool(v & 1), [bool(v >> (1 + b) & 1) for b in range(L.b2h_net_layer_bottoms(self._h, i))]))
        return out

    def loss_blob(self):
        """The blob a trainer of this net reports as its loss ('' when there is none)."""
        L = lib()
        L.b2h_net_loss_blob.argtypes = [C.c_void_p, C.c_char_p, C.c_int]
        buf = C.create_string_buffer(256)
        L.b2h_net_loss_blob(self._h, buf, 256)
        return buf.value.decode()

    def uses_database(self, layer_index=0):
        """True when that Data layer's data_param.source opened and the layer will read it (else: synthetic source)."""
        L = lib()
        L.b2h_net_layer_uses_database.argtypes = [C.c_void_p, C.c_int]
        return bool(L.b2h_net_layer_uses_database(self._h, layer_index))

    def __del__(self):
        if getattr(self, "_h", None) and _lib is not None:
            _lib.b2h_net_destroy(self._h)
            self._h = None


def solver_from_prototxt(path_or_text, is_text=False, entry="b2h_solver_from_file"):
    """(SGDSolver, net_path) from a solver.prototxt of type SGD; any other type is refused (open_solver reads every type)."""
    L = lib()
    fn = getattr(L, entry)
    fn.restype = C.c_void_p
    fn.argtypes = [C.c_char_p, C.c_int, C.c_char_p, C.c_int]
    buf = C.create_string_buffer(512)
    h = fn(path_or_text.encode(), int(is_text), buf, 512)
    if not h:
        raise HostError(L.b2h_last_error().decode())
    s = SGDSolver.__new__(SGDSolver)
    s._h = h
    return s, buf.value.decode()


def open_solver(path_or_text, is_text=False):
    """(solver, net_path) from a solver.prototxt of any type: `type`, or the legacy `solver_type` enum."""
    return solver_from_prototxt(path_or_text, is_text, entry="b2h_solver_open")


def textproto_scalar(path_or_text, key, default=None, is_text=False):
    """First scalar value (as str) of a top-level field of a text-format protobuf file, or `default` when the field is absent."""
    L = lib()
    L.b2h_textproto_scalar.argtypes = [C.c_char_p, C.c_int, C.c_char_p, C.c_char_p, C.c_int]
    buf = C.create_string_buffer(1024)
    r = L.b2h_textproto_scalar(path_or_text.encode(), int(is_text), key.encode(), buf, 1024)
    if r < 0:
        raise HostError(L.b2h_last_error().decode())
    return buf.value.decode() if r else default


def solver_describe(s):
    L = lib()
    L.b2h_solver_describe.argtypes = [C.c_void_p] + [C.POINTER(C.c_float)] * 3 + [C.POINTER(C.c_int)] * 2 + [C.c_char_p, C.c_int]
    a, b, c = C.c_float(), C.c_float(), C.c_float()
    d, e = C.c_int(), C.c_int()
    pol = C.create_string_buffer(64)
    L.b2h_solver_describe(s._h, C.byref(a), C.byref(b), C.byref(c), C.byref(d), C.byref(e), pol, 64)
    L.b2h_solver_hparams.argtypes = [C.c_void_p, C.c_char_p, C.c_int] + [C.POINTER(C.c_float)] * 3
    ty, delta, m2, rho = C.create_string_buffer(64), C.c_float(), C.c_float(), C.c_float()
    L.b2h_solver_hparams(s._h, ty, 64, C.byref(delta), C.byref(m2), C.byref(rho))
    L.b2h_solver_testing.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_char_p, C.c_int]
    ti, interval, tcl, nb = (C.c_int * 64)(), C.c_int(), C.c_int(), C.create_string_buffer(256)
    n = L.b2h_solver_testing(s._h, ti, 64, C.byref(interval), C.byref(tcl), nb, 256)
    if n > 64:
        ti = (C.c_int * n)()
        L.b2h_solver_testing(s._h, ti, n, C.byref(interval), C.byref(tcl), nb, 256)
    return dict(base_lr=a.value, momentum=b.value, weight_decay=c.value, max_iter=d.value, iter_size=e.value, lr_policy=pol.value.decode(),
                type=ty.value.decode(), delta=delta.value, momentum2=m2.value, rms_decay=rho.value,
                test_iter=[ti[k] for k in range(n)], test_interval=interval.value, test_compute_loss=bool(tcl.value),
                test_fields_not_built=nb.value.decode().split())


# ---------------------------------------------------------------------------------------------- TrainNet
class Trainer:
    """caffe::TrainNet: the whole prototxt net (synthetic data source) + SGDSolver + ReduceScheduler, on the GPU."""

    def __init__(self, net, solver, batch=0, num_classes=1000, seed=1701, math=capi.MATH_FP32, net_is_text=True,
                 solver_is_text=True, default_channels=3, default_size=224):
        L = lib()
        L.b2h_trainer_create.restype = C.c_void_p
        L.b2h_trainer_create.argtypes = [C.c_char_p, C.c_int, C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_ulonglong, C.c_int, C.c_int, C.c_int]
        self._h = L.b2h_trainer_create(net.encode(), int(net_is_text), solver.encode(), int(solver_is_text), batch, num_classes, seed,
                                       math, default_channels, default_size)
        if not self._h:
            raise HostError(L.b2h_last_error().decode())
        vp, i = C.c_void_p, C.c_int
        L.b2h_trainer_destroy.argtypes = [vp]
        L.b2h_trainer_attach_sync.argtypes = [vp, i, i, C.c_char_p, i]
        L.b2h_trainer_step.argtypes = [vp, i, i]
        L.b2h_trainer_forward_backward.argtypes = [vp, C.POINTER(C.c_float)]
        L.b2h_trainer_clear_param_diffs.argtypes = [vp]
        L.b2h_trainer_bucket_timing.argtypes = [vp, C.c_int]
        L.b2h_trainer_bucket_times.argtypes = [vp, C.c_int, C.POINTER(C.c_ulonglong), C.POINTER(C.c_float), C.POINTER(C.c_int)]
        L.b2h_trainer_sync.argtypes = [vp]
        L.b2h_trainer_loss.argtypes = [vp, C.POINTER(C.c_float)]
        L.b2h_trainer_blob_count.argtypes = [vp, C.c_char_p]
        L.b2h_trainer_blob_count.restype = C.c_longlong
        L.b2h_trainer_blob.argtypes = [vp, C.c_char_p, i, i, _f32]
        L.b2h_trainer_num_params.argtypes = [vp]
        L.b2h_trainer_num_learnable.argtypes = [vp]
        L.b2h_trainer_param_count.argtypes = [vp, i]
        L.b2h_trainer_param_count.restype = C.c_longlong
        L.b2h_trainer_param.argtypes = [vp, i, i, i, _f32]
        L.b2h_trainer_activation_floats.argtypes = [vp]
        L.b2h_trainer_activation_floats.restype = C.c_longlong

    def new_unique_id(self):
        buf = C.create_string_buffer(128)
        _ck(lib().b2h_trainer_attach_sync(self._h, 1, 0, buf, 1))
        return buf.raw

    def attach_sync(self, nranks, rank, id_bytes):
        _ck(lib().b2h_trainer_attach_sync(self._h, nranks, rank, C.create_string_buffer(bytes(id_bytes), 128), 0))

    def step(self, n=1, copy_input=False):
        _ck(lib().b2h_trainer_step(self._h, n, int(copy_input)))

    def timed_steps(self, n, copy_input=False, read_loss=False):
        """n Solver::Step iterations bracketed by CUDA events on the net's stream -> milliseconds."""
        L = lib()
        L.b2h_trainer_timed_steps.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_float)]
        v = C.c_float()
        _ck(L.b2h_trainer_timed_steps(self._h, n, int(copy_input), int(read_loss), C.byref(v)))
        return v.value

    def input_bytes(self):
        L = lib()
        L.b2h_trainer_input_bytes.argtypes = [C.c_void_p]
        L.b2h_trainer_input_bytes.restype = C.c_longlong
        return L.b2h_trainer_input_bytes(self._h)

    def forward_backward(self):
        v = C.c_float()
        _ck(lib().b2h_trainer_forward_backward(self._h, C.byref(v)))
        return v.value

    def bucket_timing(self, on):
        _ck(lib().b2h_trainer_bucket_timing(self._h, 1 if on else 0))

    def bucket_times(self, cap=4096):
        """[(bytes, ms)] of every bucket allreduce since bucket_timing(True), in issue order; drains the comm stream."""
        by = (C.c_ulonglong * cap)()
        ms = (C.c_float * cap)()
        n = C.c_int()
        _ck(lib().b2h_trainer_bucket_times(self._h, cap, by, ms, C.byref(n)))
        return [(int(by[i]), float(ms[i])) for i in range(min(n.value, cap))]

    def clip_state(self):
        """(norm, factor, clipped_count) with clip_gradients: the last step's L2 norm of the gradient, the factor the update used,
        and the steps clipped so far.  Synchronises the device."""
        return _clip_state(lib().b2h_trainer_clip_state, self._h)

    def clear_param_diffs(self):
        """Net::ClearParamDiffs: Step() expects zeroed diffs (the update clears them); call this after a forward_backward() made
        for inspection."""
        _ck(lib().b2h_trainer_clear_param_diffs(self._h))

    def sync(self):
        _ck(lib().b2h_trainer_sync(self._h))

    def loss(self):
        v = C.c_float()
        _ck(lib().b2h_trainer_loss(self._h, C.byref(v)))
        return v.value

    def get_blob(self, name, diff=False):
        n = lib().b2h_trainer_blob_count(self._h, name.encode())
        if n < 0:
            raise HostError("no blob " + name)
        out = np.empty(n, np.float32)
        _ck(lib().b2h_trainer_blob(self._h, name.encode(), int(diff), 0, out))
        return out

    def set_blob(self, name, arr, diff=False):
        _ck(lib().b2h_trainer_blob(self._h, name.encode(), int(diff), 1, np.ascontiguousarray(arr, np.float32).reshape(-1)))

    def num_params(self):
        """Blobs the layers differentiate (weights, biases, BatchNorm scale / bias); the index space of get/set_param."""
        return lib().b2h_trainer_num_params(self._h)

    def num_learnable(self):
        """Net::learnable_params() of the reference: every layer blob (BatchNorm contributes 5), = SolverState history length."""
        return lib().b2h_trainer_num_learnable(self._h)

    def get_param(self, i, what=0):
        """what: 0 data, 1 diff, 2 history, 3 second history (AdaDelta, Adam)."""
        out = np.empty(lib().b2h_trainer_param_count(self._h, i), np.float32)
        _ck(lib().b2h_trainer_param(self._h, i, what, 0, out))
        return out

    def set_param(self, i, arr, what=0):
        _ck(lib().b2h_trainer_param(self._h, i, what, 1, np.ascontiguousarray(arr, np.float32).reshape(-1)))

    def activation_floats(self):
        return lib().b2h_trainer_activation_floats(self._h)

    def layer_blob_pointers(self, layer, blob):
        """(Blob object address, device data pointer, device diff pointer) of blob `blob` of layer `layer` (execution order)"""
        L = lib()
        u = C.c_ulonglong
        L.b2h_trainer_layer_blob.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(u), C.POINTER(u), C.POINTER(u)]
        o, d, g = u(), u(), u()
        _ck(L.b2h_trainer_layer_blob(self._h, layer, blob, C.byref(o), C.byref(d), C.byref(g)))
        return o.value, d.value, g.value

    def database_batches(self):
        """Batches the LMDB-backed Data layer has loaded so far, or -1 when the net runs on the synthetic source."""
        L = lib()
        L.b2h_trainer_database_batches.argtypes = [C.c_void_p]
        L.b2h_trainer_database_batches.restype = C.c_longlong
        return L.b2h_trainer_database_batches(self._h)

    def arena_floats(self):
        """Elements of the contiguous parameter arena (= the buffer the gradient allreduce covers)."""
        L = lib()
        L.b2h_trainer_arena_floats.argtypes = [C.c_void_p]
        L.b2h_trainer_arena_floats.restype = C.c_longlong
        return L.b2h_trainer_arena_floats(self._h)

    def layers(self):
        """[(name, type)] of the net's layers in execution order."""
        L = lib()
        L.b2h_trainer_num_layers.argtypes = [C.c_void_p]
        L.b2h_trainer_layer.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_char_p, C.c_int]
        out = []
        for i in range(L.b2h_trainer_num_layers(self._h)):
            a, b = C.create_string_buffer(256), C.create_string_buffer(256)
            _ck(L.b2h_trainer_layer(self._h, i, a, b, 256))
            out.append((a.value.decode(), b.value.decode()))
        return out

    def profile(self, nsteps=2):
        """Mean ms per step of every layer call: [(layer index, op, ms)], op in fwd / bwd / wgrad / dgrad (the last two are the
        conv layers' weight- and data-gradient calls, nested inside their bwd)."""
        L = lib()
        L.b2h_trainer_profile.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_float), C.POINTER(C.c_int)]
        cap = 8192
        la, op, ms, n = (C.c_int * cap)(), (C.c_int * cap)(), (C.c_float * cap)(), C.c_int()
        _ck(L.b2h_trainer_profile(self._h, nsteps, cap, la, op, ms, C.byref(n)))
        names = ("fwd", "bwd", "wgrad", "dgrad")
        return [(la[i], names[op[i]], float(ms[i])) for i in range(min(n.value, cap))]

    def snapshot(self, prefix):
        """Solver::Snapshot: writes <prefix>_iter_<N>.caffemodel and .solverstate; returns the .solverstate path."""
        L = lib()
        L.b2h_trainer_snapshot.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_int]
        buf = C.create_string_buffer(1024)
        _ck(L.b2h_trainer_snapshot(self._h, prefix.encode(), buf, 1024))
        return buf.value.decode()

    def restore(self, solverstate_path):
        L = lib()
        L.b2h_trainer_restore.argtypes = [C.c_void_p, C.c_char_p]
        _ck(L.b2h_trainer_restore(self._h, solverstate_path.encode()))

    def copy_trained_layers_from(self, caffemodel_path):
        L = lib()
        L.b2h_trainer_copy_from.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_int)]
        n = C.c_int()
        _ck(L.b2h_trainer_copy_from(self._h, caffemodel_path.encode(), C.byref(n)))
        return n.value

    def iter(self):
        L = lib()
        L.b2h_trainer_iter.argtypes = [C.c_void_p]
        return L.b2h_trainer_iter(self._h)

    def __del__(self):
        if getattr(self, "_h", None) and _lib is not None:
            _lib.b2h_trainer_destroy(self._h)
            self._h = None


# ---------------------------------------------------------------------------------------------- TEST-phase net
class Tester:
    """A TEST-phase net (the prototxt filtered for phase TEST) run forward only: BatchNorm on its running statistics, Dropout the
    identity, Data layers on the centre crop window.  Weights come from a .caffemodel (copy_trained_layers_from) or are shared with a
    live Trainer (share_trained_layers_with), and test(k) scores k batches like the reference's `caffe test`."""

    def __init__(self, net, batch=0, num_classes=1000, seed=1701, math=capi.MATH_FP32, net_is_text=True, default_channels=3,
                 default_size=224):
        L = lib()
        vp, i = C.c_void_p, C.c_int
        L.b2h_tester_create.restype = vp
        L.b2h_tester_create.argtypes = [C.c_char_p, i, i, i, C.c_ulonglong, i, i, i]
        for fn in ("b2h_tester_destroy", "b2h_tester_forward", "b2h_tester_num_outputs", "b2h_tester_has_solver", "b2h_tester_num_layers"):
            getattr(L, fn).argtypes = [vp]
        L.b2h_tester_copy_from.argtypes = [vp, C.c_char_p, C.POINTER(i)]
        L.b2h_tester_share_from.argtypes = [vp, vp]
        L.b2h_tester_output.argtypes = [vp, i, C.c_char_p, i, C.POINTER(C.c_float), C.POINTER(C.c_longlong)]
        L.b2h_tester_test.argtypes = [vp, i, _f32, _f32, C.POINTER(C.c_float)]
        L.b2h_tester_blob_count.argtypes = [vp, C.c_char_p]
        L.b2h_tester_blob_count.restype = C.c_longlong
        L.b2h_tester_blob.argtypes = [vp, C.c_char_p, i, _f32]
        L.b2h_tester_layer.argtypes = [vp, i, C.c_char_p, C.c_char_p, i]
        L.b2h_tester_timed_forwards.argtypes = [vp, i, C.POINTER(C.c_float)]
        L.b2h_tester_profile.argtypes = [vp, i, i, C.POINTER(i), C.POINTER(C.c_float), C.POINTER(i)]
        L.b2h_tester_database_batches.argtypes = [vp]
        L.b2h_tester_database_batches.restype = C.c_longlong
        self._trainer = None
        self._h = L.b2h_tester_create(net.encode(), int(net_is_text), batch, num_classes, seed, math, default_channels, default_size)
        if not self._h:
            raise HostError(L.b2h_last_error().decode())

    def copy_trained_layers_from(self, caffemodel_path):
        """Net::CopyTrainedLayersFrom: layers matched by name; returns the number of layers copied."""
        n = C.c_int()
        _ck(lib().b2h_tester_copy_from(self._h, caffemodel_path.encode(), C.byref(n)))
        return n.value

    def share_trained_layers_with(self, trainer):
        """Net::ShareTrainedLayersWith: read `trainer`'s parameter blobs (and BatchNorm statistics) in place from now on."""
        _ck(lib().b2h_tester_share_from(self._h, trainer._h))
        self._trainer = trainer                    # the shared blobs live in the trainer's arena

    def forward(self):
        _ck(lib().b2h_tester_forward(self._h))

    def outputs(self):
        """[(name, loss_weight, count)] of the net's output blobs, in the reference's (name) order."""
        out = []
        for i in range(lib().b2h_tester_num_outputs(self._h)):
            nm, w, n = C.create_string_buffer(256), C.c_float(), C.c_longlong()
            _ck(lib().b2h_tester_output(self._h, i, nm, 256, C.byref(w), C.byref(n)))
            out.append((nm.value.decode(), w.value, n.value))
        return out

    def test(self, iterations):
        """(per_batch [iterations x output elements], means [output elements], mean loss), like tools/caffe.cpp test()."""
        width = sum(n for _, _, n in self.outputs())
        per_batch, mean, loss = np.empty(iterations * width, np.float32), np.empty(max(width, 1), np.float32), C.c_float()
        _ck(lib().b2h_tester_test(self._h, iterations, per_batch, mean, C.byref(loss)))
        return per_batch.reshape(iterations, width), mean[:width], loss.value

    def test_pass(self, iterations, between=None):
        """Solver::Test's pass: (means [output elements], loss) of `iterations` batches, scores summed on the device -- and over the
        ranks when the tester shares a trainer with an attached sync -- and read once at the end.  means = sum / batches / ranks, the
        float sums of test(); loss = sum of loss_weight * mean.  between(i), if given, is called before batch i; a false return stops the
        pass and test_pass returns None.  (On several ranks every rank must run the whole pass.)"""
        L = lib()
        hook_t = C.CFUNCTYPE(C.c_int, C.c_int)
        L.b2h_tester_test_pass.argtypes = [C.c_void_p, C.c_int, _f32, C.POINTER(C.c_float), hook_t]
        width = sum(n for _, _, n in self.outputs())
        mean, loss = np.empty(max(width, 1), np.float32), C.c_float()
        hook = hook_t(lambda i: 1 if between(i) else 0) if between else hook_t()
        ran = L.b2h_tester_test_pass(self._h, iterations, mean, C.byref(loss), hook)
        if ran < 0:
            raise HostError(L.b2h_last_error().decode())
        return (mean[:width], loss.value) if ran == iterations else None

    def get_blob(self, name):
        n = lib().b2h_tester_blob_count(self._h, name.encode())
        if n < 0:
            raise HostError("no blob " + name)
        out = np.empty(n, np.float32)
        _ck(lib().b2h_tester_blob(self._h, name.encode(), 0, out))
        return out

    def set_blob(self, name, arr):
        _ck(lib().b2h_tester_blob(self._h, name.encode(), 1, np.ascontiguousarray(arr, np.float32).reshape(-1)))

    def has_solver(self):
        return bool(lib().b2h_tester_has_solver(self._h))

    def layers(self):
        out = []
        for i in range(lib().b2h_tester_num_layers(self._h)):
            a, b = C.create_string_buffer(256), C.create_string_buffer(256)
            _ck(lib().b2h_tester_layer(self._h, i, a, b, 256))
            out.append((a.value.decode(), b.value.decode()))
        return out

    def timed_forwards(self, n):
        """n TEST forwards bracketed by CUDA events on the net's stream -> milliseconds."""
        v = C.c_float()
        _ck(lib().b2h_tester_timed_forwards(self._h, n, C.byref(v)))
        return v.value

    def profile(self, n=2):
        """[(layer index, mean forward ms)] over n forwards, CUDA events around every layer call."""
        cap = 8192
        la, ms, cnt = (C.c_int * cap)(), (C.c_float * cap)(), C.c_int()
        _ck(lib().b2h_tester_profile(self._h, n, cap, la, ms, C.byref(cnt)))
        return [(la[i], float(ms[i])) for i in range(min(cnt.value, cap))]

    def database_batches(self):
        return lib().b2h_tester_database_batches(self._h)

    def __del__(self):
        if getattr(self, "_h", None) and _lib is not None:
            _lib.b2h_tester_destroy(self._h)
            self._h = None

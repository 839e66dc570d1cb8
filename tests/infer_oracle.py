"""CPU oracle of the TEST phase for the inference tests: BatchNorm on its running statistics (the reference's TEST branch,
batch_norm_layer.cu:22-34 + :80-90), a TEST-mode forward over tests/netoracle.py's layer specs (Dropout the identity, Accuracy,
loss weights), and .caffemodel files written / read through the host layer's wire format.  TEST INFRASTRUCTURE ONLY."""
import ctypes as C

import numpy as np

import oracle
from oracle import layers_oracle as lo
import netoracle as no


def bn_forward_inference(x, gamma, beta, eps, run_mean, run_var, residual=None, relu=False):
    """y = [relu]((x - mean) * (run_var + eps)^-1/2 [* gamma + beta] [+ residual]).  run_var holds variance + eps already (the TRAIN
    side adds eps before the running average), and the TEST branch adds eps again: both are kept."""
    f = np.float32
    shp = (1, -1) + (1,) * (x.ndim - 2)
    invstd = (f(1) / np.sqrt(run_var.astype(f) + f(eps))).astype(f)
    y = ((x.astype(f) - run_mean.astype(f).reshape(shp)) * invstd.reshape(shp)).astype(f)
    if gamma is not None:          # one rounding, like the kernel's fused multiply-add
        y = (y.astype(np.float64) * gamma.reshape(shp) + beta.reshape(shp)).astype(f)
    if residual is not None:
        y = (y + residual.astype(f)).astype(f)
    return np.maximum(y, f(0)) if relu else y


def forward_test_phase(spec, params, stats, data, label, eps=1e-4):
    """The TEST-phase forward of a netoracle spec: params in no.param_shapes order, stats = {bn layer: (running mean, running var)}.
    Returns the dict of blob values; loss layers store their scalar under their top name."""
    v, pi = {"data": data, "label": label}, 0
    for L in spec:
        t, n = L["t"], L["n"]
        if t == "conv":
            w = params[pi]; pi += 1
            b = None
            if L.get("bias"):
                b = params[pi]; pi += 1
            v[n] = oracle.conv_forward(L["prm"], v[L["b"]], w, b)
        elif t == "bn":
            v[n] = bn_forward_inference(v[L["b"]], params[pi], params[pi + 1], eps, *stats[n])
            pi += 2
        elif t == "relu":
            v[L["b"]] = lo.relu_forward(v[L["b"]])
        elif t == "pool":
            v[n], _ = lo.pool_forward(v[L["b"]], no.POOL[L["m"]], (L["k"],) * 2, (L["s"],) * 2, (L["p"],) * 2)
        elif t == "sum":
            v[n] = v[L["b"][0]] + v[L["b"][1]]
        elif t == "fc":
            v[n] = lo.ip_forward(v[L["b"]], params[pi], params[pi + 1])
            pi += 2
        elif t == "loss":
            _, v[L.get("top", n)] = lo.softmax_loss_forward(v[L["b"][0]], label)
        elif t == "lrn":
            v[n], _ = lo.lrn_forward(v[L["b"]], L["size"], L["alpha"], L["beta"], L["k"])
        elif t == "concat":
            v[n] = np.concatenate([v[b] for b in L["b"]], axis=1)
        # dropout: the identity in TEST
    return v


def model_layers(spec, params, stats):
    """[(layer name, type, [blobs])] of a .caffemodel for the spec: conv w (, b); BatchNorm mean, variance, correction, scale, shift;
    InnerProduct w, b (the blob order of the layers' blobs_)."""
    out, pi = [], 0
    for L in spec:
        t, n = L["t"], L["n"]
        if t == "conv":
            k = 2 if L.get("bias") else 1
            out.append((n, "Convolution", params[pi:pi + k])); pi += k
        elif t == "bn":
            m, var = stats[n]
            out.append((n, "BatchNorm", [m, var, np.ones(1, np.float32), params[pi], params[pi + 1]])); pi += 2
        elif t == "fc":
            out.append((n, "InnerProduct", params[pi:pi + 2])); pi += 2
    return out


def _wire(lib):
    vp, i = C.c_void_p, C.c_int
    lib.b2h_wire_new.restype = vp
    lib.b2h_wire_destroy.argtypes = [vp]
    lib.b2h_wire_add_layer.argtypes = [vp, C.c_char_p, C.c_char_p]
    lib.b2h_wire_add_blob.argtypes = [vp, i, i, C.POINTER(i), C.POINTER(C.c_float)]
    lib.b2h_wire_save_model.argtypes = [vp, C.c_char_p, C.c_char_p, i]
    lib.b2h_wire_load.restype = vp
    lib.b2h_wire_load.argtypes = [C.c_char_p, i]
    lib.b2h_wire_num_layers.argtypes = [vp]
    lib.b2h_wire_layer.argtypes = [vp, i, C.c_char_p, C.c_char_p, i, C.POINTER(i)]
    lib.b2h_wire_blob.argtypes = [vp, i, i, C.POINTER(i), C.POINTER(i), C.POINTER(C.c_longlong), C.c_void_p]
    return lib


def write_caffemodel(lib, path, layers, name="mini"):
    L = _wire(lib)
    h = L.b2h_wire_new()
    try:
        for nm, ty, blobs in layers:
            li = L.b2h_wire_add_layer(h, nm.encode(), ty.encode())
            for b in blobs:
                b = np.ascontiguousarray(b, np.float32)
                shp = (C.c_int * max(b.ndim, 1))(*(b.shape or (1,)))
                assert L.b2h_wire_add_blob(h, li, max(b.ndim, 1), shp, b.ctypes.data_as(C.POINTER(C.c_float))) == 0
        assert L.b2h_wire_save_model(h, path.encode(), name.encode(), 1) == 0
    finally:
        L.b2h_wire_destroy(h)


def read_caffemodel(lib, path):
    """{layer name: [blobs as float32 arrays]}"""
    L = _wire(lib)
    h = L.b2h_wire_load(path.encode(), 0)
    assert h, lib.b2h_last_error().decode()
    out = {}
    try:
        for i in range(L.b2h_wire_num_layers(h)):
            nm, ty, nb = C.create_string_buffer(256), C.create_string_buffer(256), C.c_int()
            L.b2h_wire_layer(h, i, nm, ty, 256, C.byref(nb))
            blobs = []
            for j in range(nb.value):
                nd, shp, cnt = C.c_int(), (C.c_int * 8)(), C.c_longlong()
                L.b2h_wire_blob(h, i, j, C.byref(nd), shp, C.byref(cnt), None)
                a = np.empty(cnt.value, np.float32)
                L.b2h_wire_blob(h, i, j, C.byref(nd), shp, C.byref(cnt), a.ctypes.data_as(C.c_void_p))
                blobs.append(a.reshape([shp[k] for k in range(nd.value)]))
            out[nm.value.decode()] = blobs
    finally:
        L.b2h_wire_destroy(h)
    return out


def random_model(spec, rng):
    """Random parameters (no.param_shapes order) and non-trivial running statistics for every BatchNorm layer of the spec."""
    params, stats, chan = [], {}, {}
    for _, kind, shp in no.param_shapes(spec):
        if kind == "w":
            params.append((rng.standard_normal(shp) * np.sqrt(2.0 / np.prod(shp[1:]))).astype(np.float32))
        elif kind == "scale":
            params.append(rng.uniform(0.5, 1.5, shp).astype(np.float32))
        else:
            params.append(rng.uniform(-0.2, 0.2, shp).astype(np.float32))
    for name, kind, shp in no.param_shapes(spec):
        if kind == "scale":
            stats[name] = (rng.uniform(-0.5, 0.5, shp).astype(np.float32), rng.uniform(0.5, 2.0, shp).astype(np.float32))
    return params, stats

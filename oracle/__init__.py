"""CPU oracle loader -- TEST INFRASTRUCTURE ONLY.

ctypes bindings over ``oracle/libb2o.so`` (the plain-C restatement of the reference's
CPU conv / im2col / GEMM / SGD / allreduce path, ``oracle/b2o_oracle.c``) and, when
present, ``oracle/_ref/libb2o_ref.so`` (the reference's own ``src/caffe/util/im2col.cpp``
compiled verbatim + an OpenBLAS-driven conv loop).

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may import this package.  The product package
``caffe_mpi_b200`` never does.
"""
import ctypes as C
import glob
import os
import subprocess
import sys

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_f32p = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")
_i32p = np.ctypeslib.ndpointer(dtype=np.int32, flags="C_CONTIGUOUS")


class ConvParams(C.Structure):
    """Mirror of b2o_conv_params / ref_conv_params (same field order)."""
    _fields_ = [(n, C.c_int) for n in
                ("N", "C", "H", "W", "O", "G", "kh", "kw", "sh", "sw", "ph", "pw", "dh", "dw", "has_bias")]

    @classmethod
    def make(cls, N, Cin, H, W, O, k, s=1, p=0, d=1, G=1, bias=True):
        kh, kw = (k, k) if isinstance(k, int) else k
        sh, sw = (s, s) if isinstance(s, int) else s
        ph, pw = (p, p) if isinstance(p, int) else p
        dh, dw = (d, d) if isinstance(d, int) else d
        return cls(N, Cin, H, W, O, G, kh, kw, sh, sw, ph, pw, dh, dw, int(bool(bias)))

    @property
    def Ho(self):
        return (self.H + 2 * self.ph - (self.dh * (self.kh - 1) + 1)) // self.sh + 1

    @property
    def Wo(self):
        return (self.W + 2 * self.pw - (self.dw * (self.kw - 1) + 1)) // self.sw + 1

    @property
    def Kd(self):
        return (self.C // self.G) * self.kh * self.kw

    def x_shape(self):
        return (self.N, self.C, self.H, self.W)

    def w_shape(self):
        return (self.O, self.C // self.G, self.kh, self.kw)

    def y_shape(self):
        return (self.N, self.O, self.Ho, self.Wo)

    def flops(self):
        """2*N*O*(C/g)*kh*kw*Ho*Wo (SURVEY 8d), one pass."""
        return 2 * self.N * self.O * self.Kd * self.Ho * self.Wo


def build(force=False):
    so = os.path.join(_HERE, "libb2o.so")
    src = os.path.join(_HERE, "b2o_oracle.c")
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "libb2o.so"], stdout=subprocess.DEVNULL)
    if os.path.isdir("/root/reference/src/caffe/util"):
        ref = os.path.join(_HERE, "_ref", "libb2o_ref.so")
        drv = os.path.join(_HERE, "ref_driver.cpp")
        if force or not os.path.exists(ref) or os.path.getmtime(ref) < os.path.getmtime(drv):
            subprocess.check_call(["make", "-C", _HERE, "ref"], stdout=subprocess.DEVNULL)
    return so


_lib = None
_ref = None


def lib():
    global _lib
    if _lib is None:
        so = build()
        L = C.CDLL(so)
        P = C.POINTER(ConvParams)
        L.b2o_im2col.argtypes = [_f32p] + [C.c_int] * 11 + [_f32p]
        L.b2o_col2im.argtypes = [_f32p] + [C.c_int] * 11 + [_f32p]
        L.b2o_im2col_nd.argtypes = [_f32p, C.c_int] + [_i32p] * 6 + [_f32p]
        L.b2o_col2im_nd.argtypes = [_f32p, C.c_int] + [_i32p] * 6 + [_f32p]
        L.b2o_gemm.argtypes = [C.c_int] * 5 + [C.c_float, _f32p, _f32p, C.c_float, _f32p, C.c_int]
        L.b2o_gemv.argtypes = [C.c_int] * 3 + [C.c_float, _f32p, _f32p, C.c_float, _f32p, C.c_int]
        L.b2o_gemm_ffma.argtypes = [C.c_int] * 5 + [C.c_float, _f32p, _f32p, C.c_float, _f32p, _f32p]
        L.b2o_gemv_ffma.argtypes = [C.c_int] * 3 + [C.c_float, _f32p, _f32p, C.c_float, _f32p, _f32p]
        L.b2o_conv_forward.argtypes = [P, _f32p, _f32p, C.c_void_p, _f32p, C.c_int]
        L.b2o_conv_backward.argtypes = [P, _f32p, _f32p, _f32p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        L.b2o_conv_direct.argtypes = [P, _f32p, _f32p, C.c_void_p, _f32p]
        L.b2o_conv_fwd_ffma.argtypes = [P, _f32p, _f32p, C.c_void_p, _f32p]
        L.b2o_conv_dgrad_ffma.argtypes = [P, _f32p, _f32p, _f32p]
        L.b2o_conv_wgrad_ffma.argtypes = [P, _f32p, _f32p, _f32p]
        L.b2o_sgd_update.argtypes = [C.c_size_t, _f32p, _f32p, _f32p, C.c_float, C.c_float, C.c_float,
                                     C.c_int, C.c_float, C.c_int, C.c_int]
        L.b2o_learning_rate.argtypes = [C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_int, C.c_int,
                                        C.c_float, C.c_int, C.c_int, C.c_float]
        L.b2o_learning_rate.restype = C.c_float
        L.b2o_allreduce_avg.argtypes = [C.c_int, C.c_size_t, C.POINTER(C.c_void_p), C.c_int]
        L.b2o_momentum.argtypes = [C.c_int, C.c_int, C.c_float, C.c_float, C.c_int, C.c_float, C.c_int, C.c_float]
        L.b2o_momentum.restype = C.c_float
        L.b2o_solver_fp32.argtypes = [C.c_int, C.c_uint, C.c_size_t, _f32p, _f32p, _f32p, _f32p, _f32p, C.c_float,
                                      C.c_float, C.c_int, C.c_float, C.c_int]
        _f64p = np.ctypeslib.ndpointer(np.float64, flags="C_CONTIGUOUS")
        L.b2o_solver_f64.argtypes = [C.c_int, C.c_size_t, _f32p, _f32p, _f32p, _f32p, _f32p, C.c_float, C.c_float, C.c_int,
                                     C.c_float, C.c_int, _f64p, _f64p]
        _lib = L
    return _lib


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


# ----------------------------------------------------------------------------- numpy-level API
def im2col(im, k, s=1, p=0, d=1):
    Cc, H, W = im.shape
    prm = ConvParams.make(1, Cc, H, W, 1, k, s, p, d)
    col = np.empty((Cc * prm.kh * prm.kw, prm.Ho, prm.Wo), np.float32)
    lib().b2o_im2col(np.ascontiguousarray(im, np.float32), Cc, H, W, prm.kh, prm.kw, prm.ph, prm.pw,
                     prm.sh, prm.sw, prm.dh, prm.dw, col)
    return col


def col2im(col, im_shape, k, s=1, p=0, d=1):
    Cc, H, W = im_shape
    prm = ConvParams.make(1, Cc, H, W, 1, k, s, p, d)
    im = np.empty((Cc, H, W), np.float32)
    lib().b2o_col2im(np.ascontiguousarray(col, np.float32), Cc, H, W, prm.kh, prm.kw, prm.ph, prm.pw,
                     prm.sh, prm.sw, prm.dh, prm.dw, im)
    return im


def _nd_shapes(im_shape, k, s, p, d):
    nax = len(im_shape) - 1
    k, s, p, d = (np.asarray(v, np.int32) for v in (k, s, p, d))
    out = [(im_shape[1 + a] + 2 * p[a] - (d[a] * (k[a] - 1) + 1)) // s[a] + 1 for a in range(nax)]
    col_shape = np.asarray([im_shape[0] * int(np.prod(k))] + out, np.int32)
    return nax, np.asarray(im_shape, np.int32), col_shape, k, p, s, d


def im2col_nd(im, k, s, p, d):
    nax, ims, cols, k, p, s, d = _nd_shapes(im.shape, k, s, p, d)
    col = np.empty(tuple(cols), np.float32)
    lib().b2o_im2col_nd(np.ascontiguousarray(im, np.float32), nax, ims, cols, k, p, s, d, col)
    return col


def col2im_nd(col, im_shape, k, s, p, d):
    nax, ims, cols, k, p, s, d = _nd_shapes(im_shape, k, s, p, d)
    im = np.empty(tuple(im_shape), np.float32)
    lib().b2o_col2im_nd(np.ascontiguousarray(col, np.float32), nax, ims, cols, k, p, s, d, im)
    return im


def gemm(transA, transB, M, N, K, alpha, A, B, beta, Cm, acc64=False):
    Cm = np.ascontiguousarray(Cm, np.float32).copy()
    lib().b2o_gemm(int(transA), int(transB), M, N, K, alpha, np.ascontiguousarray(A, np.float32).ravel(),
                   np.ascontiguousarray(B, np.float32).ravel(), beta, Cm.reshape(-1), int(acc64))
    return Cm


def gemv(transA, M, N, alpha, A, x, beta, y, acc64=False):
    y = np.ascontiguousarray(y, np.float32).copy()
    lib().b2o_gemv(int(transA), M, N, alpha, np.ascontiguousarray(A, np.float32).ravel(),
                   np.ascontiguousarray(x, np.float32), beta, y, int(acc64))
    return y


def gemm_ffma(transA, transB, M, N, K, alpha, A, B, beta, Cm):
    """What the product's FFMA GEMM kernel (sgemm_simt_kernel) stores, bit for bit: an array [3, M, N] of the admissible results
    (the three ways alpha * acc + beta * c may be contracted; all equal when beta == 0).  A, B: op(A) is M x K, op(B) K x N in
    the row-major layouts b2c_sgemm takes; Cm: C before the call."""
    out = np.empty((3, M, N), np.float32)
    lib().b2o_gemm_ffma(int(transA), int(transB), M, N, K, alpha, np.ascontiguousarray(A, np.float32).reshape(-1),
                        np.ascontiguousarray(B, np.float32).reshape(-1), beta, np.ascontiguousarray(Cm, np.float32).reshape(-1),
                        out.reshape(-1))
    return out


def gemv_ffma(transA, M, N, alpha, A, x, beta, y):
    """What the product's FFMA GEMV kernels store, bit for bit: [3, len(y)] admissible results, as gemm_ffma.  A is M x N."""
    n = N if transA else M
    out = np.empty((3, n), np.float32)
    lib().b2o_gemv_ffma(int(transA), M, N, alpha, np.ascontiguousarray(A, np.float32).reshape(-1),
                        np.ascontiguousarray(x, np.float32).reshape(-1), beta, np.ascontiguousarray(y, np.float32).reshape(-1),
                        out.reshape(-1))
    return out


def ffma_match(got, admissible):
    """mask of the elements of `got` equal, bit for bit (int32 views: a zero's sign counts), to one of the admissible results"""
    g = np.ascontiguousarray(got, np.float32).view(np.int32)
    a = np.ascontiguousarray(admissible, np.float32).view(np.int32)
    return (g == a[0]) | (g == a[1]) | (g == a[2])


def conv_forward(prm, x, w, bias=None, acc64=False):
    y = np.empty(prm.y_shape(), np.float32)
    lib().b2o_conv_forward(C.byref(prm), np.ascontiguousarray(x, np.float32), np.ascontiguousarray(w, np.float32),
                           _ptr(bias), y, int(acc64))
    return y


def conv_backward(prm, x, w, dy, dw=None, db=None, want_dx=True, acc64=False):
    """dw / db are accumulated into copies of the arrays passed (or zeros); returns (dw, db, dx)."""
    dw = np.zeros(prm.w_shape(), np.float32) if dw is None else np.ascontiguousarray(dw, np.float32).copy()
    if prm.has_bias:
        db = np.zeros((prm.O,), np.float32) if db is None else np.ascontiguousarray(db, np.float32).copy()
    else:
        db = None
    dx = np.empty(prm.x_shape(), np.float32) if want_dx else None
    lib().b2o_conv_backward(C.byref(prm), np.ascontiguousarray(x, np.float32), np.ascontiguousarray(w, np.float32),
                            np.ascontiguousarray(dy, np.float32), _ptr(dw), _ptr(db), _ptr(dx), int(acc64))
    return dw, db, dx


def conv_direct(prm, x, w, bias=None):
    y = np.empty(prm.y_shape(), np.float32)
    lib().b2o_conv_direct(C.byref(prm), np.ascontiguousarray(x, np.float32), np.ascontiguousarray(w, np.float32),
                          _ptr(bias), y)
    return y


def conv_fwd_ffma(prm, x, w, bias=None):
    """What the product's FFMA forward kernel (conv_fwd_simt_kernel) stores, bit for bit: one fmaf chain per output over
    (c, i, j) without the padded taps, then + bias"""
    y = np.empty(prm.y_shape(), np.float32)
    lib().b2o_conv_fwd_ffma(C.byref(prm), np.ascontiguousarray(x, np.float32), np.ascontiguousarray(w, np.float32),
                            _ptr(None if bias is None else np.ascontiguousarray(bias, np.float32)), y)
    return y


def conv_dgrad_ffma(prm, w, dy):
    """What the product's FFMA data-gradient kernel (conv_dgrad_simt_kernel) stores, bit for bit: one fmaf chain per dx element
    over (i, j, o in the group), on-grid taps only"""
    dx = np.empty(prm.x_shape(), np.float32)
    lib().b2o_conv_dgrad_ffma(C.byref(prm), np.ascontiguousarray(dy, np.float32), np.ascontiguousarray(w, np.float32), dx)
    return dx


def conv_wgrad_ffma(prm, x, dy, dw0=None):
    """What the product's FFMA weight-gradient kernel (conv_wgrad_simt_kernel) leaves in dw, bit for bit, starting from dw0
    (zeros when None): 256 lane-strided chains, the warp butterflies, the 8 warp partials in order, one add onto dw0"""
    dw = np.zeros(prm.w_shape(), np.float32) if dw0 is None else np.ascontiguousarray(dw0, np.float32).reshape(prm.w_shape()).copy()
    lib().b2o_conv_wgrad_ffma(C.byref(prm), np.ascontiguousarray(x, np.float32), np.ascontiguousarray(dy, np.float32), dw)
    return dw


def sgd_update(g, w, h, momentum, local_rate, local_decay, l2=True, grad_scale=1.0, iter_size=1, clear_grads=True):
    g, w, h = (np.ascontiguousarray(a, np.float32).copy().reshape(-1) for a in (g, w, h))
    lib().b2o_sgd_update(g.size, g, w, h, momentum, local_rate, local_decay, int(l2), grad_scale, iter_size,
                         int(clear_grads))
    return g, w, h


LR_POLICIES = {"fixed": 0, "step": 1, "exp": 2, "inv": 3, "multistep": 4, "poly": 5, "sigmoid": 6}


def learning_rate(policy, it, base_lr, gamma=0.0, power=0.0, stepsize=1, max_iter=1, min_lr=0.0, current_step=0,
                  rampup_interval=0, rampup_lr=0.0):
    return float(lib().b2o_learning_rate(LR_POLICIES[policy], it, base_lr, gamma, power, stepsize, max_iter, min_lr,
                                         current_step, rampup_interval, rampup_lr))


MOMENTUM_POLICIES = {"fixed": 0, "poly": 1, "opt": 2}


def momentum(policy, it, momentum, max_momentum=0.99, has_max_momentum=False, momentum_power=1.0, max_iter=1, lr=0.0):
    """SGDSolver::GetMomentum at iteration `it`; lr: the learning rate at `it` ("opt")"""
    return float(lib().b2o_momentum(MOMENTUM_POLICIES[policy], it, momentum, max_momentum, int(has_max_momentum),
                                    momentum_power, max_iter, lr))


# b2c_solver_kind, and the form bits b2o_solver_fp32 reads for each
SOLVER_KINDS = {"SGD": 0, "Nesterov": 1, "AdaGrad": 2, "RMSProp": 3, "AdaDelta": 4, "Adam": 5}
_FORM_BITS = {"SGD": 4, "Nesterov": 6, "AdaGrad": 3, "RMSProp": 4, "AdaDelta": 7, "Adam": 6}


def solver_forms(kind):
    """every admissible `form` of solver_fp32 for `kind`: at most one fused product per a*b + c*d site"""
    return [f for f in range(1 << _FORM_BITS[kind]) if all((f >> b) & 3 != 3 for b in (0, 2, 4))]


def _hp_array(hp):
    return np.array([hp.get("momentum", 0.0), hp.get("delta", 1e-8), hp.get("rms_decay", 0.0), hp.get("beta1", 0.9),
                     hp.get("beta2", 0.999)], np.float32)


def _solver_inputs(g, w, h, h2):
    g, w, h = (np.ascontiguousarray(a, np.float32).reshape(-1).copy() for a in (g, w, h))
    h2 = np.zeros_like(h) if h2 is None else np.ascontiguousarray(h2, np.float32).reshape(-1).copy()
    return g, w, h, h2


def solver_fp32(kind, form, g, w, h, h2, hp, lr, decay, l2=True, grad_scale=1.0, clear_grads=True):
    """what the fused solver kernel (sgd.cu) stores for `kind` under contraction `form` (solver_forms), bit for bit:
    (g, w, h, h2) after the update.  hp: dict of momentum, delta (unclamped), rms_decay, beta1, beta2; for Adam, lr carries
    the bias correction.  h2 may be None for the one-history kinds (then returned unchanged as zeros)."""
    g, w, h, h2 = _solver_inputs(g, w, h, h2)
    rc = lib().b2o_solver_fp32(SOLVER_KINDS[kind], form, g.size, g, w, h, h2, _hp_array(hp), lr, decay, int(l2), grad_scale,
                               int(clear_grads))
    if rc:
        raise ValueError(f"form {form:#x} is not admissible for {kind}")
    return g, w, h, h2


def solver_f64(kind, g, w, h, h2, hp, lr, decay, l2=True, grad_scale=1.0, clear_grads=True):
    """the same update in float64 from the same fp32 inputs: (vals, bounds), each [4, n] for g, w, h, h2, where bounds[k][i]
    bounds |fp32 result - vals| for every admissible form (derivation at b2o_solver_f64 in b2o_oracle.c)"""
    g, w, h, h2 = _solver_inputs(g, w, h, h2)
    vals, bounds = np.empty((4, g.size)), np.empty((4, g.size))
    lib().b2o_solver_f64(SOLVER_KINDS[kind], g.size, g, w, h, h2, _hp_array(hp), lr, decay, int(l2), grad_scale,
                         int(clear_grads), vals.reshape(-1), bounds.reshape(-1))
    return vals, bounds


def allreduce_avg(bufs, solver_count=None):
    bufs = [np.ascontiguousarray(b, np.float32).copy() for b in bufs]
    arr = (C.c_void_p * len(bufs))(*[b.ctypes.data for b in bufs])
    lib().b2o_allreduce_avg(len(bufs), bufs[0].size, arr, solver_count or len(bufs))
    return bufs


# ----------------------------------------------------------------------------- reference-compiled leg
def ref():
    """oracle/_ref/libb2o_ref.so (reference im2col.cpp verbatim + OpenBLAS conv loop) or None."""
    global _ref
    if _ref is None:
        build()
        so = os.path.join(_HERE, "_ref", "libb2o_ref.so")
        if not os.path.exists(so):
            return None
        R = C.CDLL(so)
        R.ref_im2col_cpu.argtypes = [_f32p] + [C.c_int] * 11 + [_f32p]
        R.ref_col2im_cpu.argtypes = [_f32p] + [C.c_int] * 11 + [_f32p]
        R.ref_im2col_nd_cpu.argtypes = [_f32p, C.c_int] + [_i32p] * 6 + [_f32p]
        R.ref_col2im_nd_cpu.argtypes = [_f32p, C.c_int] + [_i32p] * 6 + [_f32p]
        R.ref_blas_open.argtypes = [C.c_char_p, C.c_int]
        R.ref_conv_fwd_bwd.argtypes = [C.POINTER(ConvParams), _f32p, _f32p] + [C.c_void_p] * 6
        _ref = R
    return _ref


def find_openblas():
    """The LP64 OpenBLAS shipped in the venv (SURVEY 8c); None if absent."""
    pats = [os.path.join(p, "opencv_python_headless.libs", "libopenblas*.so*") for p in sys.path if p]
    for pat in pats:
        hits = sorted(glob.glob(pat))
        if hits:
            return hits[0]
    return None


def ref_blas_open(threads=0):
    R = ref()
    path = find_openblas()
    if R is None or path is None:
        return False
    # the wheel-bundled OpenBLAS needs its sibling libquadmath / libgfortran resolved first
    d = os.path.dirname(path)
    for dep in ("libquadmath*", "libgfortran*"):
        for hit in sorted(glob.glob(os.path.join(d, dep))):
            try:
                C.CDLL(hit, mode=C.RTLD_GLOBAL)
            except OSError:
                pass
    return R.ref_blas_open(path.encode(), threads or (os.cpu_count() or 1)) == 0


def ref_conv_fwd_bwd(prm, x, w, bias, y=None, dy=None, dw=None, db=None, dx=None):
    return ref().ref_conv_fwd_bwd(C.byref(prm), x, w, _ptr(bias), _ptr(y), _ptr(dy), _ptr(dw), _ptr(db), _ptr(dx))

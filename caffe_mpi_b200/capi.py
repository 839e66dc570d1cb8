"""ctypes binding of include/b2c.h (one-to-one; no logic beyond argument marshalling)."""
import ctypes as C
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libb2c.so")
HEADER = os.path.join(os.path.dirname(_HERE), "include", "b2c.h")

ENGINE_DEFAULT, ENGINE_CAFFE, ENGINE_CUDNN = 0, 1, 2
MATH_FP32, MATH_TF32, MATH_FP32_3XTF32 = 0, 1, 2
ALGO_AUTO, ALGO_SIMT, ALGO_TCGEN05 = 0, 1, 2
OP_FORWARD, OP_BACKWARD_DATA, OP_BACKWARD_FILTER = 0, 1, 2
UNIQUE_ID_BYTES = 128
# b2c_wgrad_route, in enum order
WGRAD_ROUTES = ("caffe", "simt", "gather", "staged_3x3", "staged_3x3_plane", "staged_1x1", "staged_1x1_plane", "tma_1x1",
                "compact_staged", "compact_tma")
# b2c_conv_route, in enum order
CONV_ROUTES = ("caffe", "simt", "gather", "gather_scatter", "staged", "staged_plane")
# b2c_pool_route, in enum order
POOL_ROUTES = ("max_scalar", "max_window", "max_bwd_row", "max_bwd_quad", "ave")
# b2c_sgemm_route, in enum order
SGEMM_ROUTES = ("ffma", "tc")
# b2c_deconv_route, in enum order
DECONV_ROUTES = ("dual", "phase", "depthwise")
# b2c_softmax_loss_route and b2c_loss_normalization, in enum order
SOFTMAX_LOSS_ROUTES = ("row", "column", "column_f4")
LOSS_NORMS = ("FULL", "VALID", "BATCH_SIZE", "NONE")
# b2c_neuron_kind, in enum order
NEURON_KINDS = ("ELU", "POWER", "ABSVAL", "BNLL", "EXP", "LOG", "THRESHOLD")


class B2CError(RuntimeError):
    pass


class ConvParams(C.Structure):
    """b2c_conv_params."""
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
        return 2 * self.N * self.O * self.Kd * self.Ho * self.Wo


class DetectNetAug(C.Structure):
    """b2c_detectnet_aug: one image's augmentation (the reference's AugmentSelection)."""
    _fields_ = [("hue_rotation", C.c_float), ("saturation", C.c_float), ("flip", C.c_int), ("scale_w", C.c_int), ("scale_h", C.c_int),
                ("rotation", C.c_float), ("crop_x", C.c_int), ("crop_y", C.c_int)]


DETECTNET_MAX_CLASSES = 32
DETECTNET_BAD_BOX_LENGTH, DETECTNET_TOO_MANY_BOXES = 1, 2
GRIDBOX_TYPES = ("GRIDBOX_MAX", "GRIDBOX_MIN")


class DetectNetGT(C.Structure):
    """b2c_detectnet_gt: DetectNetGroundTruthParameter with RECTANGULAR coverage."""
    _fields_ = [(n, C.c_int) for n in ("image_size_x", "image_size_y", "stride", "gridbox_type", "max_cvg_len", "min_cvg_len",
                                      "obj_norm", "crop_bboxes")] + \
               [("scale_cvg", C.c_float), ("n_classes", C.c_int), ("class_src", C.c_int * DETECTNET_MAX_CLASSES),
                ("class_dst", C.c_int * DETECTNET_MAX_CLASSES)]

    @classmethod
    def make(cls, image_size_x=1248, image_size_y=384, stride=4, gridbox_type="GRIDBOX_MAX", max_cvg_len=50, min_cvg_len=50,
             obj_norm=False, crop_bboxes=True, scale_cvg=0.5, object_class=()):
        """caffe.proto's defaults; object_class a sequence of (src, dst) (empty: the reference's {1 -> 0})."""
        g = cls(image_size_x, image_size_y, stride, GRIDBOX_TYPES.index(gridbox_type) if isinstance(gridbox_type, str) else gridbox_type,
                max_cvg_len, min_cvg_len, int(bool(obj_norm)), int(bool(crop_bboxes)), scale_cvg, len(object_class))
        for m, (src, dst) in enumerate(object_class):
            g.class_src[m], g.class_dst[m] = src, dst
        return g


def declared_symbols():
    """Every function name include/b2c.h declares."""
    txt = open(HEADER).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(b2c_[a-z0-9_]+)\s*\(", txt)))


_lib = None


def lib():
    """Load libb2c.so (built in-tree by __graft_entry__.build()).  Fails loudly if it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_SO):
        raise B2CError(f"{_SO} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                       "(there is no CPU or PyTorch fallback for this path)")
    try:
        import torch  # noqa: F401  (loads the CUDA runtime + NCCL this process will share)
    except Exception:  # pragma: no cover
        pass
    L = C.CDLL(_SO, mode=C.RTLD_GLOBAL)
    vp, i, f, sz = C.c_void_p, C.c_int, C.c_float, C.c_size_t
    P = C.POINTER(ConvParams)
    sig = {
        "b2c_last_error": (C.c_char_p, []),
        "b2c_version": (C.c_char_p, []),
        "b2c_launch_count": (C.c_uint64, []),
        "b2c_set_default_math": (i, [i]),
        "b2c_set_default_algo": (i, [i]),
        "b2c_conv_desc_create": (i, [P, i, C.POINTER(vp)]),
        "b2c_conv_desc_destroy": (i, [vp]),
        "b2c_conv_desc_set_math": (i, [vp, i]),
        "b2c_conv_desc_set_algo": (i, [vp, i]),
        "b2c_conv_out_shape": (i, [vp, C.POINTER(i), C.POINTER(i)]),
        "b2c_conv_workspace_bytes": (sz, [vp, i]),
        "b2c_conv_algo_used": (i, [vp, i]),
        "b2c_debug_wgrad_plan": (i, [vp, C.POINTER(i), i]),
        "b2c_debug_conv_plan": (i, [vp, i, C.POINTER(i), i]),
        "b2c_conv_forward": (i, [vp, vp, vp, vp, vp, vp, sz, vp]),
        "b2c_conv_backward_data": (i, [vp, vp, vp, vp, vp, sz, vp]),
        "b2c_conv_backward_filter": (i, [vp, vp, vp, vp, vp, sz, vp]),
        "b2c_conv_wgrad_split_bytes": (sz, [vp]),
        "b2c_conv_backward_filter_split": (i, [vp, vp, vp, vp, vp, sz, vp, sz, vp]),
        "b2c_conv_backward_bias": (i, [vp, vp, vp, vp]),
        "b2c_im2col": (i, [vp] + [i] * 11 + [vp, vp]),
        "b2c_col2im": (i, [vp] + [i] * 11 + [vp, vp]),
        "b2c_im2col_nd": (i, [vp, i] + [C.POINTER(i)] * 6 + [vp, vp]),
        "b2c_col2im_nd": (i, [vp, i] + [C.POINTER(i)] * 6 + [vp, vp]),
        "b2c_sgemm": (i, [i, i, i, i, i, f, vp, vp, f, vp, vp]),
        "b2c_sgemv": (i, [i, i, i, f, vp, vp, f, vp, vp]),
        "b2c_sgemm_workspace_bytes": (sz, [i, i, i, i, i]),
        "b2c_sgemm_tc_supported": (i, [i, i, i, i, i]),
        "b2c_transpose": (i, [i, i, vp, vp, vp]),
        "b2c_sgemm_ex": (i, [i, i, i, i, i, f, vp, vp, f, vp, vp, sz, vp]),
        "b2c_debug_sgemm_plan": (i, [i, i, i, i, i, f, f, vp, vp, vp, sz, C.POINTER(i), i]),
        "b2c_sgd_update": (i, [sz, vp, vp, vp, f, f, f, i, f, i, vp]),
        "b2c_sgd_update_arena": (i, [i, C.POINTER(sz), C.POINTER(sz), C.POINTER(f), C.POINTER(f), vp, vp, vp,
                                     f, i, f, i, vp]),
        "b2c_solver_update_arena": (i, [i, i, C.POINTER(sz), C.POINTER(sz), C.POINTER(f), C.POINTER(f), vp, vp, vp, vp,
                                        SolverHParams, i, f, i, vp]),
        "b2c_debug_solver_plan": (i, [i, i, C.POINTER(sz), C.POINTER(sz), vp, vp, vp, vp, C.POINTER(i), i, C.POINTER(i),
                                      C.POINTER(C.c_longlong)]),
        "b2c_arena_sumsq": (i, [i, C.POINTER(sz), C.POINTER(sz), C.POINTER(sz), vp, vp, vp]),
        "b2c_clip_factor": (i, [vp, sz, C.c_double, f, vp, vp]),
        "b2c_solver_update_arena_scaled": (i, [i, i, C.POINTER(sz), C.POINTER(sz), C.POINTER(f), C.POINTER(f), vp, vp, vp, vp,
                                               SolverHParams, i, f, vp, i, vp]),
        "b2c_debug_sumsq_plan": (i, [i, C.POINTER(sz), C.POINTER(sz), C.POINTER(sz), vp, C.POINTER(i), i, C.POINTER(i),
                                     C.POINTER(C.c_longlong), C.POINTER(C.c_longlong)]),
        "b2c_relu_forward": (i, [sz, vp, vp, f, vp]),
        "b2c_relu_backward": (i, [sz, vp, vp, vp, f, vp]),
        "b2c_bn_forward_train": (i, [i, i, i, vp, vp, vp, f, f, i, vp, vp, vp, vp, vp, vp, vp]),
        "b2c_bn_backward": (i, [i, i, i, vp, vp, vp, vp, vp, vp, vp, vp]),
        "b2c_bn_forward_train_fused": (i, [i, i, i, vp, vp, vp, f, f, i, vp, vp, vp, vp, vp, i, vp]),
        "b2c_bn_backward_fused": (i, [i, i, i, vp, vp, vp, vp, vp, vp, vp, vp, vp, i, vp]),
        "b2c_bn_forward_train_fused_res": (i, [i, i, i, vp, vp, vp, f, f, i, vp, vp, vp, vp, vp, vp, i, vp]),
        "b2c_bn_backward_fused_res": (i, [i, i, i, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
        "b2c_add_relu": (i, [sz, vp, vp, vp, vp]),
        "b2c_relu_backward2": (i, [sz, vp, vp, vp, vp, vp]),
        "b2c_pool_forward": (i, [i] * 10 + [vp, vp, vp, vp]),
        "b2c_pool_backward": (i, [i] * 10 + [vp, vp, vp, vp]),
        "b2c_debug_pool_plan": (i, [i] * 11 + [vp, vp, C.POINTER(i), i]),
        "b2c_debug_bn_plan": (i, [i] * 5 + [C.POINTER(vp), i, C.POINTER(i), i]),
        "b2c_add": (i, [sz, vp, vp, vp, vp]),
        "b2c_softmax_loss_forward": (i, [i, i, vp, vp, vp, vp, vp]),
        "b2c_softmax_loss_backward": (i, [i, i, vp, vp, f, vp, vp]),
        "b2c_softmax_loss_workspace": (i, [i, i, i, C.POINTER(sz)]),
        "b2c_softmax_loss_forward_ex": (i, [i, i, i, vp, vp, i, i, i, vp, vp, vp, vp, vp]),
        "b2c_softmax_loss_backward_ex": (i, [i, i, i, vp, vp, i, i, vp, f, vp, vp]),
        "b2c_debug_softmax_loss_plan": (i, [i, i, i, vp, vp, C.POINTER(i), i]),
        "b2c_accuracy_ex": (i, [i, i, i, i, vp, vp, i, i, vp, vp, vp, vp]),
        "b2c_softmax_forward": (i, [i, i, i, vp, vp, vp]),
        "b2c_softmax_backward": (i, [i, i, i, vp, vp, vp, vp]),
        "b2c_sigmoid_forward": (i, [sz, vp, vp, vp]),
        "b2c_sigmoid_backward": (i, [sz, vp, vp, vp, vp]),
        "b2c_neuron_forward": (i, [i, sz, vp, vp, f, f, f, vp]),
        "b2c_neuron_backward": (i, [i, sz, vp, vp, vp, vp, f, f, f, vp]),
        "b2c_prelu_forward": (i, [i, i, i, i, vp, vp, vp, vp, vp]),
        "b2c_prelu_workspace_bytes": (i, [i, i, i, i, C.POINTER(sz)]),
        "b2c_prelu_backward": (i, [i, i, i, i, vp, vp, vp, vp, vp, vp, sz, vp]),
        "b2c_debug_neuron_plan": (i, [i, i, i, i, i, i, C.POINTER(vp), i, C.POINTER(i), i]),
        "b2c_sigmoid_ce_loss_forward": (i, [i, sz, vp, vp, vp, vp]),
        "b2c_sigmoid_ce_loss_backward": (i, [sz, vp, vp, f, vp, vp]),
        "b2c_euclidean_loss_forward": (i, [i, sz, vp, vp, vp, vp, vp]),
        "b2c_euclidean_loss_backward": (i, [sz, vp, f, vp, vp]),
        "b2c_l1_loss_forward": (i, [i, sz, vp, vp, vp, vp, vp]),
        "b2c_l1_loss_backward": (i, [sz, vp, f, vp, vp]),
        "b2c_detectnet_image_workspace_bytes": (sz, [i, i, i]),
        "b2c_detectnet_image": (i, [i, i, i, i, i, vp, vp, i, vp, C.POINTER(f), vp, sz, vp, vp]),
        "b2c_detectnet_label_shape": (i, [C.POINTER(DetectNetGT), C.POINTER(i), C.POINTER(i), C.POINTER(i)]),
        "b2c_detectnet_labels": (i, [i, i, i, i, vp, vp, C.POINTER(DetectNetGT), vp, vp, vp]),
        "b2c_debug_detectnet_plan": (i, [i, i, i, i, i, i, i, C.POINTER(DetectNetGT), C.POINTER(i), i]),
        "b2c_contrastive_loss_forward": (i, [i, i, vp, vp, vp, f, i, vp, vp, vp, vp]),
        "b2c_contrastive_loss_backward": (i, [i, i, vp, vp, vp, f, i, f, vp, vp, vp]),
        "b2c_bias_forward": (i, [i, i, i, vp, vp, vp]),
        "b2c_bias_backward": (i, [i, i, i, vp, vp, vp]),
        "b2c_lrn_forward": (i, [i, i, i, i, f, f, f, vp, vp, vp, vp]),
        "b2c_lrn_backward": (i, [i, i, i, i, f, f, vp, vp, vp, vp, vp, vp]),
        "b2c_dropout_mask": (i, [sz, f, C.c_ulonglong, C.c_ulonglong, vp, vp]),
        "b2c_mul": (i, [sz, vp, vp, vp, vp]),
        "b2c_deconv_desc_create": (i, [P, i, C.POINTER(vp)]),
        "b2c_deconv_desc_destroy": (i, [vp]),
        "b2c_deconv_desc_set_math": (i, [vp, i]),
        "b2c_deconv_desc_set_algo": (i, [vp, i]),
        "b2c_deconv_out_shape": (i, [vp, C.POINTER(i), C.POINTER(i)]),
        "b2c_deconv_workspace_bytes": (sz, [vp, i]),
        "b2c_deconv_forward": (i, [vp, vp, vp, vp, vp, vp, sz, vp]),
        "b2c_deconv_backward_data": (i, [vp, vp, vp, vp, vp, sz, vp]),
        "b2c_deconv_backward_filter": (i, [vp, vp, vp, vp, vp, sz, vp]),
        "b2c_deconv_wgrad_split_bytes": (sz, [vp]),
        "b2c_deconv_backward_filter_split": (i, [vp, vp, vp, vp, vp, sz, vp, sz, vp]),
        "b2c_deconv_backward_bias": (i, [vp, vp, vp, vp]),
        "b2c_debug_deconv_plan": (i, [vp, i, C.POINTER(i), i]),
        "b2c_crop_forward": (i, [i, C.POINTER(i), C.POINTER(i), C.POINTER(i), vp, vp, vp]),
        "b2c_crop_backward": (i, [i, C.POINTER(i), C.POINTER(i), C.POINTER(i), vp, vp, vp]),
        "b2c_comm_get_unique_id": (i, [vp]),
        "b2c_comm_init": (i, [i, i, vp, C.POINTER(vp)]),
        "b2c_comm_destroy": (i, [vp]),
        "b2c_comm_nranks": (i, [vp]),
        "b2c_comm_bcast": (i, [vp, vp, sz, i, vp]),
        "b2c_comm_allreduce_sum": (i, [vp, vp, sz, vp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = res, args
    _lib = L
    return L


def check(rc):
    if rc != 0:
        raise B2CError(f"b2c error {rc}: {lib().b2c_last_error().decode()}")


def _p(t):
    """device pointer of a torch tensor (or None)."""
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream(stream=None):
    import torch
    s = stream if stream is not None else torch.cuda.current_stream()
    return C.c_void_p(s.cuda_stream)


class ConvDesc:
    """b2c_conv_desc owner; methods take torch CUDA tensors and forward raw pointers to the C ABI."""

    def __init__(self, params, engine=ENGINE_DEFAULT, math=None, algo=None):
        self.params = params
        self.engine = engine
        h = C.c_void_p()
        check(lib().b2c_conv_desc_create(C.byref(params), engine, C.byref(h)))
        self._h = h
        if math is not None:
            check(lib().b2c_conv_desc_set_math(h, math))
        if algo is not None:
            check(lib().b2c_conv_desc_set_algo(h, algo))
        self._ws = None

    def __del__(self):
        if getattr(self, "_h", None) and _lib is not None:
            _lib.b2c_conv_desc_destroy(self._h)
            self._h = None

    def workspace_bytes(self, op):
        return int(lib().b2c_conv_workspace_bytes(self._h, op))

    def algo_used(self, op):
        return int(lib().b2c_conv_algo_used(self._h, op))

    def wgrad_plan(self):
        """b2c_debug_wgrad_plan: the weight-gradient route for 16-byte aligned operands and its split-K plan."""
        out = (C.c_int * 7)()
        check(lib().b2c_debug_wgrad_plan(self._h, out, 7))
        return dict(route=WGRAD_ROUTES[out[0]], splits=out[1], per=out[2], nkb=out[3], cols=out[4], bpi=out[5],
                    presplit_dy=bool(out[6]))

    def conv_plan(self, op):
        """b2c_debug_conv_plan: the forward (op 0) or data-gradient (op 1) route for 16-byte aligned activations and its tile
        plan; `variant` is the gather kernel's KMODE or the staged kernel's box width BWT."""
        out = (C.c_int * 8)()
        check(lib().b2c_debug_conv_plan(self._h, op, out, 8))
        return dict(route=CONV_ROUTES[out[0]], n_tile=out[1], m_tiles=out[2], n_tiles=out[3], tiles=out[4], grid=out[5],
                    nkb=out[6], variant=out[7])

    def _workspace(self, op, like):
        import torch
        need = self.workspace_bytes(op)
        if need == 0:
            return None, 0
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.uint8, device=like.device)
        return C.c_void_p(self._ws.data_ptr()), self._ws.numel()

    def forward(self, x, w, bias, y, stream=None):
        ws, n = self._workspace(OP_FORWARD, x)
        check(lib().b2c_conv_forward(self._h, _p(x), _p(w), _p(bias), _p(y), ws, n, _stream(stream)))
        return y

    def backward_data(self, dy, w, dx, stream=None):
        ws, n = self._workspace(OP_BACKWARD_DATA, dy)
        check(lib().b2c_conv_backward_data(self._h, _p(dy), _p(w), _p(dx), ws, n, _stream(stream)))
        return dx

    def backward_data_accumulate_supported(self):
        return bool(lib().b2c_conv_backward_data_accumulate_supported(self._h))

    def backward_data_accumulate(self, dy, w, dx, stream=None):
        """dx += bottom gradient (the fan-out accumulation of Net::Backward folded into the kernel's TMA reduce-add store)."""
        ws, n = self._workspace(OP_BACKWARD_DATA, dy)
        check(lib().b2c_conv_backward_data_accumulate(self._h, _p(dy), _p(w), _p(dx), ws, n, _stream(stream)))
        return dx

    def backward_filter(self, x, dy, dw, stream=None):
        ws, n = self._workspace(OP_BACKWARD_FILTER, x)
        check(lib().b2c_conv_backward_filter(self._h, _p(x), _p(dy), _p(dw), ws, n, _stream(stream)))
        return dw

    def wgrad_split_bytes(self):
        return int(lib().b2c_conv_wgrad_split_bytes(self._h))

    def backward_filter_split(self, x, dy, dw, stream=None):
        """backward_filter with the split buffer of b2c_conv_wgrad_split_bytes (dY converted to bf16 hi / lo once per call)."""
        import torch
        ws, n = self._workspace(OP_BACKWARD_FILTER, x)
        need = self.wgrad_split_bytes()
        if need and (getattr(self, "_split", None) is None or self._split.numel() < need):
            self._split = torch.empty(need, dtype=torch.uint8, device=x.device)
        sp = C.c_void_p(self._split.data_ptr()) if need else None
        check(lib().b2c_conv_backward_filter_split(self._h, _p(x), _p(dy), _p(dw), ws, n, sp, need, _stream(stream)))
        return dw

    def backward_bias(self, dy, db, stream=None):
        check(lib().b2c_conv_backward_bias(self._h, _p(dy), _p(db), _stream(stream)))
        return db

    # ---- prepared filters (include/b2c.h): build the GEMM-ordered filter copies once per weight change ----
    def filter_cache_bytes(self):
        L = lib()
        L.b2c_conv_filter_cache_bytes.restype = C.c_size_t
        L.b2c_conv_filter_cache_bytes.argtypes = [C.c_void_p]
        return int(L.b2c_conv_filter_cache_bytes(self._h))

    def prepare_filter(self, w, stream=None):
        """Allocates (once) and fills the cache from `w`, binds it: forward / backward_data then skip their own prepass."""
        import torch
        need = self.filter_cache_bytes()
        if need == 0:
            return False
        if getattr(self, "_fcache", None) is None or self._fcache.numel() < need:
            self._fcache = torch.empty(need, dtype=torch.uint8, device=w.device)
        L = lib()
        L.b2c_conv_prepare_filter.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
        check(L.b2c_conv_prepare_filter(self._h, _p(w), C.c_void_p(self._fcache.data_ptr()), need, _stream(stream)))
        L.b2c_conv_desc_bind_filter_cache.argtypes = [C.c_void_p, C.c_void_p]
        check(L.b2c_conv_desc_bind_filter_cache(self._h, C.c_void_p(self._fcache.data_ptr())))
        return True

    def unbind_filter_cache(self):
        L = lib()
        L.b2c_conv_desc_bind_filter_cache.argtypes = [C.c_void_p, C.c_void_p]
        check(L.b2c_conv_desc_bind_filter_cache(self._h, None))


class DeconvDesc:
    """b2c_deconv_desc owner: a transposed convolution given by its own parameters (ConvParams with Cin = bottom channels,
    O = num_output, H, W = bottom extent).  Methods take torch CUDA tensors, like ConvDesc's."""

    def __init__(self, params, engine=ENGINE_DEFAULT, math=None, algo=None):
        self.params = params
        h = C.c_void_p()
        check(lib().b2c_deconv_desc_create(C.byref(params), engine, C.byref(h)))
        self._h = h
        if math is not None:
            check(lib().b2c_deconv_desc_set_math(h, math))
        if algo is not None:
            check(lib().b2c_deconv_desc_set_algo(h, algo))
        self._ws = None
        self._split = None

    def __del__(self):
        if getattr(self, "_h", None) and _lib is not None:
            _lib.b2c_deconv_desc_destroy(self._h)
            self._h = None

    def out_shape(self):
        ht, wt = C.c_int(), C.c_int()
        check(lib().b2c_deconv_out_shape(self._h, C.byref(ht), C.byref(wt)))
        return ht.value, wt.value

    def x_shape(self):
        p = self.params
        return (p.N, p.C, p.H, p.W)

    def w_shape(self):
        p = self.params
        return (p.C, p.O // p.G, p.kh, p.kw)

    def y_shape(self):
        p = self.params
        return (p.N, p.O) + self.out_shape()

    def workspace_bytes(self, op):
        return int(lib().b2c_deconv_workspace_bytes(self._h, op))

    def plan(self, op):
        """b2c_debug_deconv_plan: route, the dual's own route (DUAL route) and, on the phase route, (taps, tiles) per phase."""
        n = 3 + 2 * self.params.sh * self.params.sw
        out = (C.c_int * n)()
        check(lib().b2c_debug_deconv_plan(self._h, op, out, n))
        ph = [(out[3 + 2 * k], out[4 + 2 * k]) for k in range(out[2])]
        return dict(route=DECONV_ROUTES[out[0]], dual_route=out[1], phases=out[2], phase_taps=[t for t, _ in ph],
                    phase_tiles=[t for _, t in ph])

    def _workspace(self, op, like):
        import torch
        need = self.workspace_bytes(op)
        if need == 0:
            return None, 0
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.uint8, device=like.device)
        return C.c_void_p(self._ws.data_ptr()), self._ws.numel()

    def forward(self, x, w, bias, y, stream=None):
        ws, n = self._workspace(OP_FORWARD, x)
        check(lib().b2c_deconv_forward(self._h, _p(x), _p(w), _p(bias), _p(y), ws, n, _stream(stream)))
        return y

    def backward_data(self, dy, w, dx, stream=None):
        ws, n = self._workspace(OP_BACKWARD_DATA, dy)
        check(lib().b2c_deconv_backward_data(self._h, _p(dy), _p(w), _p(dx), ws, n, _stream(stream)))
        return dx

    def backward_filter(self, x, dy, dw, stream=None):
        ws, n = self._workspace(OP_BACKWARD_FILTER, x)
        check(lib().b2c_deconv_backward_filter(self._h, _p(x), _p(dy), _p(dw), ws, n, _stream(stream)))
        return dw

    def wgrad_split_bytes(self):
        return int(lib().b2c_deconv_wgrad_split_bytes(self._h))

    def backward_filter_split(self, x, dy, dw, stream=None):
        import torch
        ws, n = self._workspace(OP_BACKWARD_FILTER, x)
        need = self.wgrad_split_bytes()
        if need and (self._split is None or self._split.numel() < need):
            self._split = torch.empty(need, dtype=torch.uint8, device=x.device)
        sp = C.c_void_p(self._split.data_ptr()) if need else None
        check(lib().b2c_deconv_backward_filter_split(self._h, _p(x), _p(dy), _p(dw), ws, n, sp, need, _stream(stream)))
        return dw

    def backward_bias(self, dy, db, stream=None):
        check(lib().b2c_deconv_backward_bias(self._h, _p(dy), _p(db), _stream(stream)))
        return db


def crop_forward(bottom, top, offsets, stream=None):
    """b2c_crop_forward: top = bottom[offsets : offsets + top.shape] (offsets over every axis)."""
    nax = bottom.dim()
    check(lib().b2c_crop_forward(nax, _iarr(bottom.shape), _iarr(top.shape), _iarr(offsets), _p(bottom), _p(top), _stream(stream)))
    return top


def crop_backward(top_diff, bottom_diff, offsets, stream=None):
    """b2c_crop_backward: bottom_diff = 0, then the top diff copied into the window."""
    nax = bottom_diff.dim()
    check(lib().b2c_crop_backward(nax, _iarr(bottom_diff.shape), _iarr(top_diff.shape), _iarr(offsets), _p(top_diff),
                                  _p(bottom_diff), _stream(stream)))
    return bottom_diff


def im2col(im, col, k, s, p, d, stream=None):
    Cc, H, W = im.shape
    check(lib().b2c_im2col(_p(im), Cc, H, W, k[0], k[1], p[0], p[1], s[0], s[1], d[0], d[1], _p(col), _stream(stream)))
    return col


def col2im(col, im, k, s, p, d, stream=None):
    Cc, H, W = im.shape
    check(lib().b2c_col2im(_p(col), Cc, H, W, k[0], k[1], p[0], p[1], s[0], s[1], d[0], d[1], _p(im), _stream(stream)))
    return im


def _iarr(v):
    return (C.c_int * len(v))(*[int(a) for a in v])


def im2col_nd(im, col, k, s, p, d, stream=None):
    nax = im.dim() - 1
    check(lib().b2c_im2col_nd(_p(im), nax, _iarr(im.shape), _iarr(col.shape), _iarr(k), _iarr(p), _iarr(s), _iarr(d),
                              _p(col), _stream(stream)))
    return col


def col2im_nd(col, im, k, s, p, d, stream=None):
    nax = im.dim() - 1
    check(lib().b2c_col2im_nd(_p(col), nax, _iarr(im.shape), _iarr(col.shape), _iarr(k), _iarr(p), _iarr(s), _iarr(d),
                              _p(im), _stream(stream)))
    return im


def pool_plan(method, dir, NC, H, W, k, s, p, out_ptr=0, mask_ptr=0):
    """b2c_debug_pool_plan: the kernel b2c_pool_forward (dir 0) or b2c_pool_backward (dir 1) takes for these arguments, with y / dx
    at address out_ptr and the MAX mask at mask_ptr (integers; never dereferenced).  k, s, p: (h, w) pairs.  Raises B2CError
    where the entry points refuse the arguments."""
    out = (C.c_int * 5)()
    check(lib().b2c_debug_pool_plan(method, dir, NC, H, W, k[0], k[1], s[0], s[1], p[0], p[1], C.c_void_p(out_ptr),
                                    C.c_void_p(mask_ptr), out, 5))
    return dict(route=POOL_ROUTES[out[0]], Ho=out[1], Wo=out[2], q=out[3], rpb=out[4])


BN_FORMS = ("unfused", "fused", "fused_res")


def softmax_loss_plan(outer, Cc, inner, logits_ptr=0, prob_ptr=0):
    """b2c_debug_softmax_loss_plan: the forward route of b2c_softmax_loss_forward_ex with logits / prob at these addresses, the
    pixels per chunk, the chunks and the workspace bytes."""
    out = (C.c_int * 4)()
    check(lib().b2c_debug_softmax_loss_plan(outer, Cc, inner, C.c_void_p(logits_ptr), C.c_void_p(prob_ptr), out, 4))
    return {"route": SOFTMAX_LOSS_ROUTES[out[0]], "chunk": out[1], "slots": out[2], "workspace": out[3]}


def softmax_loss_workspace(outer, Cc, inner):
    n = C.c_size_t()
    check(lib().b2c_softmax_loss_workspace(outer, Cc, inner, C.byref(n)))
    return n.value


def softmax_loss_forward_ex(outer, Cc, inner, logits, labels, prob, loss, normalizer, workspace, ignore_label=None,
                            norm="VALID", stream=None):
    """b2c_softmax_loss_forward_ex on torch CUDA tensors; ignore_label None = not set; norm one of LOSS_NORMS."""
    check(lib().b2c_softmax_loss_forward_ex(outer, Cc, inner, _p(logits), _p(labels), int(ignore_label is not None),
                                            int(ignore_label or 0), LOSS_NORMS.index(norm), _p(prob), _p(loss), _p(normalizer),
                                            _p(workspace), _stream(stream)))


def softmax_loss_backward_ex(outer, Cc, inner, prob, labels, normalizer, loss_weight, dx, ignore_label=None, stream=None):
    check(lib().b2c_softmax_loss_backward_ex(outer, Cc, inner, _p(prob), _p(labels), int(ignore_label is not None),
                                             int(ignore_label or 0), _p(normalizer), loss_weight, _p(dx), _stream(stream)))


def accuracy_ex(outer, Cc, inner, top_k, scores, labels, accuracy, per_class, scratch, ignore_label=None, stream=None):
    """b2c_accuracy_ex; per_class may be None; scratch holds 8 + 8 * Cc bytes (8 without per_class)."""
    check(lib().b2c_accuracy_ex(outer, Cc, inner, top_k, _p(scores), _p(labels), int(ignore_label is not None), int(ignore_label or 0),
                                _p(accuracy), _p(per_class), _p(scratch), _stream(stream)))


def neuron_forward(kind, x, y, p=(0.0, 0.0, 0.0), stream=None):
    """b2c_neuron_forward on torch CUDA tensors; kind one of NEURON_KINDS; p the kind's (p0, p1, p2)."""
    p = tuple(p) + (0.0,) * (3 - len(p))
    check(lib().b2c_neuron_forward(NEURON_KINDS.index(kind), x.numel(), _p(x), _p(y), *p, _stream(stream)))


def neuron_backward(kind, x, y, dy, dx, p=(0.0, 0.0, 0.0), stream=None):
    """b2c_neuron_backward; x / y may be None where the kind's rule does not read them."""
    p = tuple(p) + (0.0,) * (3 - len(p))
    check(lib().b2c_neuron_backward(NEURON_KINDS.index(kind), dy.numel(), _p(x), _p(y), _p(dy), _p(dx), *p, _stream(stream)))


def detectnet_augs(augs):
    """A CUDA uint8 tensor holding b2c_detectnet_aug[N] for `augs`: DetectNetAug structs or dicts of their fields."""
    import torch
    arr = (DetectNetAug * len(augs))(*[a if isinstance(a, DetectNetAug) else DetectNetAug(**a) for a in augs])
    return torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).cuda()


def detectnet_image_workspace_bytes(N, H, W):
    return int(lib().b2c_detectnet_image_workspace_bytes(N, H, W))


def detectnet_image(bottom, augs, top, mean_value=None, mean_image=None, workspace=None, stream=None):
    """b2c_detectnet_image: bottom [N, 3, H, W] -> top [N, 3, OH, OW] (torch CUDA float32); augs a tensor from detectnet_augs;
    mean_value 1 or 3 floats, or mean_image [3, H, W]; workspace allocated when None."""
    import torch
    N, _, H, W = bottom.shape
    OH, OW = top.shape[2], top.shape[3]
    ws_bytes = detectnet_image_workspace_bytes(N, H, W)
    if workspace is None:
        workspace = torch.empty(ws_bytes // 4, dtype=torch.float32, device=bottom.device)
    kind, mv = 0, None
    if mean_image is not None:
        kind = 2
    elif mean_value is not None:
        vals = list(mean_value) * 3 if len(mean_value) == 1 else list(mean_value)
        kind, mv = 1, (C.c_float * 3)(*vals)
    check(lib().b2c_detectnet_image(N, H, W, OH, OW, _p(bottom), _p(augs), kind, _p(mean_image), mv, _p(workspace),
                                    workspace.numel() * 4, _p(top), _stream(stream)))


def detectnet_label_shape(gt):
    """(channels, GH, GW) of the label top for a DetectNetGT."""
    c, h, w = C.c_int(), C.c_int(), C.c_int()
    check(lib().b2c_detectnet_label_shape(C.byref(gt), C.byref(c), C.byref(h), C.byref(w)))
    return c.value, h.value, w.value


def detectnet_labels(labels, H, W, augs, gt, top, status, stream=None):
    """b2c_detectnet_labels: labels [N, 1, rows, 16] of H x W images -> top [N, C, GH, GW]; status a CUDA int32 tensor of one
    element the kernel ORs its header errors into (see detectnet_check_status)."""
    N, _, rows, _ = labels.shape
    check(lib().b2c_detectnet_labels(N, rows, H, W, _p(labels), _p(augs), C.byref(gt), _p(top), _p(status), _stream(stream)))


def detectnet_check_status(status):
    """Raise the reference's CHECK message for the error bits a label call left in `status` (an int)."""
    if status & DETECTNET_BAD_BOX_LENGTH:
        raise B2CError("DetectNetTransformation label: Check failed: bboxLen == 16 (a label header's box length is not 16)")
    if status & DETECTNET_TOO_MANY_BOXES:
        raise B2CError("DetectNetTransformation label: Check failed: numOfBbox <= height (a label header lists more boxes "
                       "than the blob has rows)")


def detectnet_plan(op, N, H, W, OH=0, OW=0, rows=0, gt=None):
    """b2c_debug_detectnet_plan: op "image" or "labels"."""
    out = (C.c_int * 6)()
    check(lib().b2c_debug_detectnet_plan(("image", "labels").index(op), N, H, W, OH, OW, rows, C.byref(gt) if gt is not None else None,
                                         out, 6))
    if op == "image":
        return dict(launches=out[0], colour_ctas=out[1], sample_ctas=out[2], threads=out[3], workspace=(out[4] << 20) + out[5])
    return dict(ctas=out[0], threads=out[1], smem=out[2], channels=out[3], grid_h=out[4], grid_w=out[5])


def prelu_forward(N, Cc, dim, shared, x, slope, y, x_keep=None, stream=None):
    check(lib().b2c_prelu_forward(N, Cc, dim, int(bool(shared)), _p(x), _p(slope), _p(y), _p(x_keep), _stream(stream)))


def prelu_workspace_bytes(N, Cc, dim, shared):
    n = C.c_size_t()
    check(lib().b2c_prelu_workspace_bytes(N, Cc, dim, int(bool(shared)), C.byref(n)))
    return n.value


def prelu_backward(N, Cc, dim, shared, x, dy, slope, dx, dslope, workspace=None, stream=None):
    """b2c_prelu_backward; dx and dslope may be None; dslope is added into.  workspace: a torch uint8 / float tensor of at least
    prelu_workspace_bytes, or None when that is 0."""
    nbytes = 0 if workspace is None else workspace.numel() * workspace.element_size()
    check(lib().b2c_prelu_backward(N, Cc, dim, int(bool(shared)), _p(x), _p(dy), _p(slope), _p(dx), _p(dslope), _p(workspace), nbytes,
                                   _stream(stream)))


NEURON_PLAN_OPS = ("forward", "backward", "prelu_forward", "prelu_backward")


def neuron_plan(op, N, Cc=1, dim=1, shared=False, kind="ELU", ptrs=()):
    """b2c_debug_neuron_plan: the launch of an elementwise neuron call over N values (op "forward" / "backward") or of a PReLU call
    (op "prelu_forward" / "prelu_backward") with the call's tensor pointers (ints, None for a null one) tested for alignment only."""
    out = (C.c_int * 7)()
    arr = (C.c_void_p * max(1, len(ptrs)))(*[p or None for p in ptrs])
    check(lib().b2c_debug_neuron_plan(NEURON_PLAN_OPS.index(op), NEURON_KINDS.index(kind), N, Cc, dim, int(bool(shared)), arr, len(ptrs),
                                      out, 7))
    return dict(vec=bool(out[0]), ctas=out[1], threads=out[2], blocks_per_channel=out[3], stripe=out[4], channels=out[5],
                workspace=out[6])


def bn_plan(dir, form, N, Cc, S, ptrs=()):
    """b2c_debug_bn_plan: the launch a BatchNorm training call (dir 0 forward, 1 backward; form one of BN_FORMS) takes, with the
    call's tensor pointers (ints, None for a null one) tested for alignment only"""
    out = (C.c_int * 6)()
    arr = (C.c_void_p * max(1, len(ptrs)))(*[p or None for p in ptrs])
    check(lib().b2c_debug_bn_plan(dir, BN_FORMS.index(form), N, Cc, S, arr, len(ptrs), out, 6))
    return dict(launches=out[0], cs=out[1], threads=out[2], park=out[3], prefetch=out[4], vec=bool(out[5]))


def sgemm(transA, transB, M, N, K, alpha, A, B, beta, Cm, stream=None):
    check(lib().b2c_sgemm(int(transA), int(transB), M, N, K, alpha, _p(A), _p(B), beta, _p(Cm), _stream(stream)))
    return Cm


def sgemm_ex(transA, transB, M, N, K, alpha, A, B, beta, Cm, stream=None):
    """b2c_sgemm_ex with the scratch b2c_sgemm_workspace_bytes asks for (split-K tensor-core path for NoTrans x Trans products)."""
    import torch
    L = lib()
    nbytes = L.b2c_sgemm_workspace_bytes(int(transA), int(transB), M, N, K)
    ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=Cm.device)
    check(L.b2c_sgemm_ex(int(transA), int(transB), M, N, K, alpha, _p(A), _p(B), beta, _p(Cm), _p(ws), nbytes, _stream(stream)))
    return Cm, nbytes


def sgemm_plan(transA, transB, M, N, K, alpha, beta, A=0, B=0, workspace=0, workspace_bytes=0):
    """b2c_debug_sgemm_plan: the kernel b2c_sgemm_ex takes for these arguments, with A, B and the workspace at these addresses
    (integers; never dereferenced; 0 = null workspace)"""
    out = (C.c_int * 7)()
    check(lib().b2c_debug_sgemm_plan(int(transA), int(transB), M, N, K, alpha, beta, C.c_void_p(A), C.c_void_p(B),
                                     C.c_void_p(workspace or None), workspace_bytes, out, 7))
    return dict(route=SGEMM_ROUTES[out[0]], cols=out[1], bpi=out[2], splits=out[3], kb_per_split=out[4], m_tiles=out[5],
                n_tiles=out[6])


def sgemv(transA, M, N, alpha, A, x, beta, y, stream=None):
    check(lib().b2c_sgemv(int(transA), M, N, alpha, _p(A), _p(x), beta, _p(y), _stream(stream)))
    return y


def sgd_update(g, w, h, momentum, local_rate, local_decay, l2=True, grad_scale=1.0, clear_grads=True, stream=None):
    check(lib().b2c_sgd_update(g.numel(), _p(g), _p(w), _p(h), momentum, local_rate, local_decay, int(l2), grad_scale,
                               int(clear_grads), _stream(stream)))


def sgd_update_arena(offsets, counts, rates, decays, g, w, h, momentum, l2=True, grad_scale=1.0, clear_grads=True,
                     stream=None):
    n = len(offsets)
    check(lib().b2c_sgd_update_arena(n, (C.c_size_t * n)(*offsets), (C.c_size_t * n)(*counts),
                                     (C.c_float * n)(*rates), (C.c_float * n)(*decays), _p(g), _p(w), _p(h),
                                     momentum, int(l2), grad_scale, int(clear_grads), _stream(stream)))


SOLVER_KINDS = {"SGD": 0, "Nesterov": 1, "AdaGrad": 2, "RMSProp": 3, "AdaDelta": 4, "Adam": 5}   # b2c_solver_kind


class SolverHParams(C.Structure):
    _fields_ = [("momentum", C.c_float), ("delta", C.c_float), ("rms_decay", C.c_float), ("beta1", C.c_float),
                ("beta2", C.c_float)]


def solver_update_arena(kind, offsets, counts, rates, decays, g, w, h, h2=None, momentum=0.0, delta=1e-8, rms_decay=0.0,
                        beta1=0.9, beta2=0.999, l2=True, grad_scale=1.0, clear_grads=True, stream=None):
    """b2c_solver_update_arena: `kind` is a name of SOLVER_KINDS (or a raw b2c_solver_kind); h2 only for AdaDelta and Adam.  For Adam, `rates` carry the
    bias correction sqrt(1-beta2^t)/(1-beta1^t)."""
    n = len(offsets)
    hp = SolverHParams(momentum, delta, rms_decay, beta1, beta2)
    check(lib().b2c_solver_update_arena(SOLVER_KINDS.get(kind, kind), n, (C.c_size_t * n)(*offsets), (C.c_size_t * n)(*counts),
                                        (C.c_float * n)(*rates), (C.c_float * n)(*decays), _p(g), _p(w), _p(h),
                                        _p(h2), hp, int(l2), grad_scale, int(clear_grads),
                                        _stream(stream)))


def solver_plan(kind, offsets, counts, g, w, h, h2=0):
    """b2c_debug_solver_plan: the launches b2c_solver_update_arena makes for this layout with the arenas at addresses g, w, h, h2
    (integers; never dereferenced; 0 = null).  kind: a name of SOLVER_KINDS or a raw b2c_solver_kind.  Returns dict(launches=[(segments, blocks), ...], segs=[dict(launch, vec, blocks,
    head, body4, tail), ...]); raises B2CError where the entry points refuse the arguments."""
    n = len(offsets)
    seg = (C.c_longlong * max(1, 6 * n))()
    nl = C.c_int()
    cap = n // 96 + 2
    lo = (C.c_int * (2 * cap))()
    check(lib().b2c_debug_solver_plan(SOLVER_KINDS.get(kind, kind), n, (C.c_size_t * max(1, n))(*offsets),
                                      (C.c_size_t * max(1, n))(*counts), C.c_void_p(g or None), C.c_void_p(w or None),
                                      C.c_void_p(h or None), C.c_void_p(h2 or None), lo, cap, C.byref(nl), seg))
    keys = ("launch", "vec", "blocks", "head", "body4", "tail")
    return dict(launches=[(lo[2 * i], lo[2 * i + 1]) for i in range(nl.value)],
                segs=[dict(zip(keys, (int(v) for v in seg[6 * s:6 * s + 6]))) for s in range(n)])


def solver_update_arena_scaled(kind, offsets, counts, rates, decays, g, w, h, h2=None, factor=None, momentum=0.0, delta=1e-8,
                               rms_decay=0.0, beta1=0.9, beta2=0.999, l2=True, grad_scale=1.0, clear_grads=True, stream=None):
    """b2c_solver_update_arena_scaled: solver_update_arena with grad_scale times the float at device address `factor` (a tensor
    or an integer address)."""
    n = len(offsets)
    hp = SolverHParams(momentum, delta, rms_decay, beta1, beta2)
    fp = C.c_void_p(factor or None) if factor is None or isinstance(factor, int) else _p(factor)
    check(lib().b2c_solver_update_arena_scaled(SOLVER_KINDS.get(kind, kind), n, (C.c_size_t * n)(*offsets),
                                               (C.c_size_t * n)(*counts), (C.c_float * n)(*rates), (C.c_float * n)(*decays),
                                               _p(g), _p(w), _p(h), _p(h2), hp, int(l2), grad_scale, fp,
                                               int(clear_grads), _stream(stream)))


def arena_sumsq(offsets, counts, slots, g, partials, stream=None):
    """b2c_arena_sumsq: float64 partials of sum(g^2), one per 4096-element block, block b of segment s at slots[s] + b."""
    n = len(offsets)
    check(lib().b2c_arena_sumsq(n, (C.c_size_t * max(1, n))(*offsets), (C.c_size_t * max(1, n))(*counts),
                                (C.c_size_t * max(1, n))(*slots), _p(g), _p(partials), _stream(stream)))


CLIP_STATE_BYTES = 16      # b2c_clip_state: float norm, float factor, long long clipped


def clip_factor(partials, nslots, s_n, clip, state, stream=None):
    """b2c_clip_factor: `state` is a device buffer of CLIP_STATE_BYTES (e.g. a 4-element float32 tensor); clip_state() reads it."""
    check(lib().b2c_clip_factor(_p(partials), nslots, s_n, clip, _p(state), _stream(stream)))


def clip_state(state):
    """(norm, factor, clipped) of a b2c_clip_state held in a 4-element float32 tensor"""
    import numpy as np
    raw = state.detach().cpu().numpy().view(np.uint8)
    return float(raw[0:4].view(np.float32)[0]), float(raw[4:8].view(np.float32)[0]), int(raw[8:16].view(np.int64)[0])


def sumsq_plan(offsets, counts, slots, g):
    """b2c_debug_sumsq_plan for the diff arena at address g (an integer; never dereferenced).  Returns dict(launches=[(segments,
    blocks), ...], segs=[dict(launch, vec, blocks, slot, head, body4, tail), ...], npartials); raises B2CError where
    b2c_arena_sumsq refuses the arguments."""
    n = len(offsets)
    seg = (C.c_longlong * max(1, 7 * n))()
    nl, npart = C.c_int(), C.c_longlong()
    cap = n // 96 + 2
    lo = (C.c_int * (2 * cap))()
    check(lib().b2c_debug_sumsq_plan(n, (C.c_size_t * max(1, n))(*offsets), (C.c_size_t * max(1, n))(*counts),
                                     (C.c_size_t * max(1, n))(*slots), C.c_void_p(g or None), lo, cap, C.byref(nl), seg,
                                     C.byref(npart)))
    keys = ("launch", "vec", "blocks", "slot", "head", "body4", "tail")
    return dict(launches=[(lo[2 * i], lo[2 * i + 1]) for i in range(nl.value)],
                segs=[dict(zip(keys, (int(v) for v in seg[7 * s:7 * s + 7]))) for s in range(n)], npartials=npart.value)


class Comm:
    """b2c_comm owner.  `id_bytes` comes from rank 0's get_unique_id() carried by the caller."""

    def __init__(self, nranks, rank, id_bytes):
        h = C.c_void_p()
        buf = C.create_string_buffer(bytes(id_bytes), UNIQUE_ID_BYTES)
        check(lib().b2c_comm_init(nranks, rank, buf, C.byref(h)))
        self._h, self.nranks, self.rank = h, nranks, rank

    @staticmethod
    def get_unique_id():
        buf = C.create_string_buffer(UNIQUE_ID_BYTES)
        check(lib().b2c_comm_get_unique_id(buf))
        return buf.raw

    def bcast(self, t, root=0, stream=None):
        check(lib().b2c_comm_bcast(self._h, _p(t), t.numel(), root, _stream(stream)))

    def allreduce_sum(self, t, count=None, stream=None):
        check(lib().b2c_comm_allreduce_sum(self._h, _p(t), t.numel() if count is None else count, _stream(stream)))

    def destroy(self):
        if self._h:
            lib().b2c_comm_destroy(self._h)
            self._h = None

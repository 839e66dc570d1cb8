"""Schedule edge cases of the forward and data-gradient kernels against the float64 CPU oracle.

b2c_conv_forward and b2c_conv_backward_data pick one of several kernels (include/b2c.h, b2c_conv_route): the TMA-staged bf16x3
kernel for stride-1 "same" convolutions (csrc/conv_tc_stg.cu; box width BWT of 128 / 160 / 192 / 256 pixels, or plane mode on
7x7 maps), the gather kernel for everything else it can tabulate (csrc/conv_tc.cu; N_TILE 32 / 64 / 128, K in chunks of four
channels or per element), the strided scatter variant of the gather kernel for the data gradient of strided 1x1 layers, and the
FFMA kernels past the gather table.  Every case below states the regime it exists for as a predicate over
ConvDesc.conv_plan(0) and conv_plan(1) (b2c_debug_conv_plan, the planners the launches run), so a planner change that moves a
case off its path fails here, naming the regime, instead of silently testing something else.  Shapes are chosen for 132 SMs.

Each case runs both ops through the C ABI with a workspace full of NaN (a filter copy that leaves its K padding unwritten
shows up) and the output as a view inside a buffer prefilled with NaN whose head and tail hold a sentinel (a write past the
last image, channel or group shows up in the guard bands, an element never written shows up as NaN):
  * parity with the oracle at the 1e-4 blob-level bar (1e-3 in TF32 math); the scatter data gradient must leave every
    off-grid element exactly 0;
  * a second call is bit-identical;
  * with a NaN-prefilled filter cache prepared and bound, the result is bit-identical to the self-contained call;
  * x (dy) and y (dx) 4 bytes off alignment: the staged layers fall back to the gather kernel (with exactly the workspace
    b2c_conv_workspace_bytes asks for and the staged filter cache bound), the gather layers take the scalar epilogue;
  * on the staged data-gradient routes, backward_data_accumulate into a random dx0 equals dx0 + the data gradient bit for bit.
The blob-level bar divides by max|ref|, so an error confined to small elements (border pixels whose taps are mostly padding, one
channel of a ragged tile) can hide under it.  The exact-integer test closes that gap: x, w, dy and the bias are integers in
[-4, 4], which bf16 and TF32 hold exactly (their lo terms are 0) and whose partial sums are integers below 2^24, so every
element of y and dx must EQUAL the oracle in every math mode.  A wrong tap mask, row wrap, flip or channel offset moves some
element by an integer.  This check cannot see a dropped lo term (lo is 0 here); test_conv_precision_gpu.py checks the lo
half of the split element by element (an exact split-term probe and a per-element error bound)."""
import ctypes as C

import numpy as np
import pytest

import oracle as o
from cases import Guarded, make, tensors, rel_err

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import caffe_mpi_b200 as m  # noqa: E402
from caffe_mpi_b200 import capi  # noqa: E402

TOL = 1e-4
STAGED = ("staged", "staged_plane")
TENSOR_CORE = STAGED + ("gather", "gather_scatter")


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


def ptr(t):
    return C.c_void_p(t.data_ptr())


def conv(N, C, H, W, O, k, s=1, p=None, d=1, G=1, bias=True):
    """p=None: "same" padding k // 2"""
    kh, kw = (k, k) if isinstance(k, int) else k
    return dict(N=N, Cin=C, H=H, W=W, O=O, k=k, s=s, p=((kh // 2, kw // 2) if p is None else p), d=d, G=G, bias=bias)


def R(q, route, **want):
    """the plan takes `route`, and every field named in `want` has that value"""
    return q["route"] == route and all(q[k] == v for k, v in want.items())


# (id, shape as a function of the SM count, regime over (forward plan, data-gradient plan, SMs), math mode, exact-integer test)
CASES = [
    # ---- staged kernel: BWT = staged pixels per channel, need = 128 + 2 * halo rounded up to 16 bytes
    ("stg_bwt128_1x1", lambda S: conv(3, 32, 8, 16, 128, 1),
     lambda q0, q1, S: R(q0, "staged", variant=128, n_tile=128) and R(q1, "staged", variant=128, n_tile=32), None, True),
    ("stg_bwt160_need_160", lambda S: conv(3, 32, 12, 15, 32, 3),                     # halo 16
     lambda q0, q1, S: R(q0, "staged", variant=160) and R(q1, "staged", variant=160), None, True),
    ("stg_bwt192_need_165_o96", lambda S: conv(3, 32, 12, 16, 96, 3),                 # halo 17: partial N_TILE 128
     lambda q0, q1, S: R(q0, "staged", variant=192, n_tile=128, n_tiles=1) and R(q1, "staged", variant=192, n_tile=32),
     None, True),
    ("stg_5x5_bwt192_o33", lambda S: conv(3, 32, 10, 14, 33, 5),                      # need 190; 31 empty columns
     lambda q0, q1, S: R(q0, "staged", variant=192, n_tile=64) and R(q1, "gather", variant=0), None, True),
    ("stg_bwt256_need_256", lambda S: conv(4, 32, 4, 63, 32, 3),                      # halo 64; 252-pixel images
     lambda q0, q1, S: R(q0, "staged", variant=256) and R(q1, "staged", variant=256), None, True),
    ("stg_need_261_gather", lambda S: conv(3, 32, 4, 64, 32, 3),
     lambda q0, q1, S: R(q0, "gather", variant=1) and R(q1, "gather", variant=1), None, True),
    ("stg_rect_1x7", lambda S: conv(3, 32, 8, 17, 32, (1, 7)),                        # halo 3
     lambda q0, q1, S: R(q0, "staged", variant=160) and R(q1, "staged", variant=160), None, True),
    ("stg_rect_7x1", lambda S: conv(3, 32, 16, 8, 32, (7, 1)),                        # halo 24
     lambda q0, q1, S: R(q0, "staged", variant=192) and R(q1, "staged", variant=192), None, True),
    ("stg_5x5_25_taps", lambda S: conv(2, 32, 8, 16, 32, 5),
     lambda q0, q1, S: R(q0, "staged", variant=256) and R(q1, "staged", variant=256), None, True),
    ("gather_7x7_49_taps", lambda S: conv(2, 32, 8, 16, 32, 7),
     lambda q0, q1, S: R(q0, "gather", variant=1) and R(q1, "gather", variant=1), None, True),
    ("stg_c48_fwd_gather_dgrad_staged", lambda S: conv(3, 48, 8, 16, 64, 3),         # dgrad: partial N_TILE 64
     lambda q0, q1, S: R(q0, "gather", variant=1) and R(q1, "staged", variant=192, n_tile=64), None, True),
    ("stg_o16_fwd_gather", lambda S: conv(3, 32, 8, 16, 16, 3),
     lambda q0, q1, S: R(q0, "gather", n_tile=32) and R(q1, "gather"), None, True),
    ("stg_o32_smallest_cout", lambda S: conv(3, 32, 8, 16, 32, 3),
     lambda q0, q1, S: R(q0, "staged", n_tile=32) and R(q1, "staged", n_tile=32), None, True),
    ("stg_map_11x13_gather", lambda S: conv(3, 32, 11, 13, 32, 3),                    # H*W % 4 != 0
     lambda q0, q1, S: R(q0, "gather") and R(q1, "gather"), None, True),
    ("stg_map_8x8_gather", lambda S: conv(3, 32, 8, 8, 32, 3),                        # H*W < 128
     lambda q0, q1, S: R(q0, "gather") and R(q1, "gather"), None, True),
    ("stg_map_7x7_plane", lambda S: conv(3, 32, 7, 7, 32, 3),
     lambda q0, q1, S: R(q0, "staged_plane", variant=49) and R(q1, "staged_plane", variant=49), None, True),
    # plane mode: 128-row tiles touch up to 4 images; the last tile has 8, 57 and 27 rows
    ("plane_1x1_o32_n8", lambda S: conv(8, 32, 7, 7, 32, 1),
     lambda q0, q1, S: R(q0, "staged_plane", m_tiles=4, n_tile=32) and R(q1, "staged_plane", m_tiles=4), None, True),
    ("plane_3x3_o72_n9", lambda S: conv(9, 32, 7, 7, 72, 3),
     lambda q0, q1, S: R(q0, "staged_plane", m_tiles=4, n_tile=128) and R(q1, "gather"), None, True),
    ("plane_5x5_o160_n11", lambda S: conv(11, 32, 7, 7, 160, 5),
     lambda q0, q1, S: R(q0, "staged_plane", m_tiles=5, n_tiles=2) and R(q1, "staged_plane", n_tile=32), None, True),
    ("stg_partial_last_tile_12x12", lambda S: conv(3, 32, 12, 12, 64, 3),             # Mtot 432
     lambda q0, q1, S: R(q0, "staged", m_tiles=4, n_tile=64) and R(q1, "staged", m_tiles=4), None, True),
    ("stg_multi_wave", lambda S: conv(2 * S + 1, 32, 8, 16, 160, 1),
     lambda q0, q1, S: R(q0, "staged", n_tiles=2) and q0["tiles"] > 2 * q0["grid"] and R(q1, "staged") and q1["tiles"] > 2 * q1["grid"],
     None, True),
    ("stg_shape_tf32", lambda S: conv(2, 32, 8, 16, 32, 3),
     lambda q0, q1, S: R(q0, "gather") and R(q1, "gather"), capi.MATH_TF32, True),
    ("stg_shape_3xtf32", lambda S: conv(2, 32, 8, 16, 32, 3),
     lambda q0, q1, S: R(q0, "gather") and R(q1, "gather"), capi.MATH_FP32_3XTF32, True),
    # ---- gather kernel
    ("g_stem_7x7_s2_kmode0", lambda S: conv(2, 3, 23, 23, 32, 7, s=2, p=3),          # K 147 padded to 160
     lambda q0, q1, S: R(q0, "gather", n_tile=32, variant=0, nkb=5) and R(q1, "simt"), None, True),
    ("g_3x3_s2_c36_nt64", lambda S: conv(2, 36, 13, 13, 64, 3, s=2, p=1),            # odd W: the right padding column is read
     lambda q0, q1, S: R(q0, "gather", n_tile=64, variant=1) and R(q1, "simt"), None, True),
    ("g_o130_ragged_nt128", lambda S: conv(2, 16, 8, 8, 130, 3),                      # second N tile: 2 columns
     lambda q0, q1, S: R(q0, "gather", n_tile=128, n_tiles=2), None, True),
    ("g_group2_og48", lambda S: conv(2, 32, 8, 8, 96, 3, G=2),                        # 16 empty columns at a group boundary
     lambda q0, q1, S: R(q0, "gather", n_tile=64, n_tiles=1, tiles=2 * q0["m_tiles"]) and R(q1, "gather", n_tile=32, variant=1),
     None, True),
    ("g_group3_cg3", lambda S: conv(2, 9, 9, 9, 24, 3, G=3),
     lambda q0, q1, S: R(q0, "gather", variant=0, tiles=3 * q0["m_tiles"]) and R(q1, "gather", variant=1), None, True),
    ("g_dilation2", lambda S: conv(2, 16, 10, 10, 32, 3, p=2, d=2),
     lambda q0, q1, S: R(q0, "gather") and R(q1, "gather"), None, True),
    ("g_dgrad_pad_minus1", lambda S: conv(2, 16, 8, 8, 32, 3, p=3),                   # dgrad pad' = 2 - 3
     lambda q0, q1, S: R(q0, "gather") and R(q1, "gather"), None, True),
    # the gather table holds 1152 entries: K / 4 chunks (KMODE 1) or padded K elements (KMODE 0)
    ("g_table_kmode1_fits", lambda S: conv(1, 512, 5, 5, 32, 3, s=2, p=1),           # K 4608
     lambda q0, q1, S: R(q0, "gather", variant=1, nkb=144), None, True),
    ("g_table_kmode1_cliff", lambda S: conv(1, 516, 5, 5, 32, 3, s=2, p=1),
     lambda q0, q1, S: R(q0, "simt"), None, True),
    ("g_table_kmode0_fits", lambda S: conv(1, 127, 5, 5, 32, 3, s=2, p=1),           # K 1143 padded to 1152
     lambda q0, q1, S: R(q0, "gather", variant=0, nkb=36), None, True),
    ("g_table_kmode0_cliff", lambda S: conv(1, 129, 5, 5, 32, 3, s=2, p=1),
     lambda q0, q1, S: R(q0, "simt"), None, True),
    ("g_table_dgrad_og512", lambda S: conv(1, 8, 4, 4, 1024, 3, G=2),
     lambda q0, q1, S: R(q0, "gather") and R(q1, "gather", variant=1, nkb=144), None, True),
    ("g_table_dgrad_og516", lambda S: conv(1, 8, 4, 4, 1032, 3, G=2),
     lambda q0, q1, S: R(q0, "gather") and R(q1, "simt"), None, True),
    # strided 1x1 data gradient: rows of the top grid scattered into a zeroed dx
    ("scatter_1x1_s2_13x13", lambda S: conv(2, 32, 13, 13, 64, 1, s=2),              # odd H, W: last row and column off-grid
     lambda q0, q1, S: R(q0, "gather") and R(q1, "gather_scatter", variant=1), None, True),
    ("scatter_1x1_s2x3", lambda S: conv(2, 32, 12, 13, 64, 1, s=(2, 3)),
     lambda q0, q1, S: R(q0, "gather") and R(q1, "gather_scatter"), None, True),
    ("scatter_1x1_s2_o33", lambda S: conv(2, 32, 14, 14, 33, 1, s=2),
     lambda q0, q1, S: R(q1, "gather_scatter", variant=0), None, True),
    # epilogues: P % 4 != 0 stores per element, P % 4 == 0 with an aligned output stores float4 (the unaligned pass of every
    # case runs the per-element path)
    ("g_epi_scalar_13x13", lambda S: conv(2, 16, 13, 13, 32, 3),
     lambda q0, q1, S: R(q0, "gather") and R(q1, "gather"), None, True),
    ("g_epi_vector_12x12", lambda S: conv(2, 16, 12, 12, 32, 3),
     lambda q0, q1, S: R(q0, "gather") and R(q1, "gather"), None, True),
    ("g_mtot_lt_128", lambda S: conv(1, 16, 5, 5, 32, 3),
     lambda q0, q1, S: R(q0, "gather", m_tiles=1) and R(q1, "gather", m_tiles=1), None, True),
    ("g_multi_wave_phase_wrap", lambda S: conv(16, 64, 56, 56, 256, 3, s=2, p=1),    # 196 tiles of 18 K blocks
     lambda q0, q1, S: R(q0, "gather", tiles=196, nkb=18) and q0["tiles"] > q0["grid"], None, False),
]
IDS = [c[0] for c in CASES]


class Run:
    """One descriptor; calls b2c_conv_forward / b2c_conv_backward_data[_accumulate] through the C ABI with a NaN-filled
    workspace of exactly b2c_conv_workspace_bytes and the output inside a Guarded buffer."""

    def __init__(self, c, math=None):
        self.c, self.po, self.pc = c, make(o, c), make(capi, c)
        self.d = m.ConvDesc(self.pc, math=math)
        self.cache = None

    def plans(self):
        return self.d.conv_plan(capi.OP_FORWARD), self.d.conv_plan(capi.OP_BACKWARD_DATA)

    def call(self, op, a, W, B=None, off=0, init=None, accumulate=False):
        """op on input `a` (x or dy, host array) with device filter W and bias B; `off`: floats of misalignment of the input
        and the output."""
        L = capi.lib()
        need = self.d.workspace_bytes(op)
        ws = torch.full((max(need, 16),), 0xFF, dtype=torch.uint8, device="cuda")
        A = torch.empty(a.size + off, device="cuda")
        A[off:] = dev(a.reshape(-1))
        shape = self.po.y_shape() if op == capi.OP_FORWARD else self.po.x_shape()
        out = Guarded(int(np.prod(shape)), off, init)
        args = (ptr(ws), C.c_size_t(need), capi._stream())
        if op == capi.OP_FORWARD:
            rc = L.b2c_conv_forward(self.d._h, ptr(A[off:]), ptr(W), None if B is None else ptr(B), out.ptr(), *args)
        elif accumulate:
            rc = L.b2c_conv_backward_data_accumulate(self.d._h, ptr(A[off:]), ptr(W), out.ptr(), *args)
        else:
            rc = L.b2c_conv_backward_data(self.d._h, ptr(A[off:]), ptr(W), out.ptr(), *args)
        capi.check(rc)
        return out.read().reshape(shape)

    def bind_cache(self, W):
        """prepare a NaN-prefilled filter cache from W and bind it; False when the layer has no cache"""
        nbytes = self.d.filter_cache_bytes()
        if not nbytes:
            return False
        self.cache = torch.full((nbytes + 256,), 0xFF, dtype=torch.uint8, device="cuda")
        base = C.c_void_p((self.cache.data_ptr() + 255) & ~255)
        L = capi.lib()
        capi.check(L.b2c_conv_prepare_filter(self.d._h, ptr(W), base, C.c_size_t(nbytes), capi._stream()))
        capi.check(L.b2c_conv_desc_bind_filter_cache(self.d._h, base))
        return True

    def unbind_cache(self):
        capi.check(capi.lib().b2c_conv_desc_bind_filter_cache(self.d._h, None))
        self.cache = None


def oracle_y(po, x, w, b):
    return o.conv_forward(po, x, w, b, acc64=True)


def oracle_dx(po, w, dy):
    """the data-gradient leg of the oracle's backward alone (null dW and db)"""
    dx = np.empty(po.x_shape(), np.float32)
    o.lib().b2o_conv_backward(C.byref(po), np.zeros(1, np.float32), np.ascontiguousarray(w, np.float32),
                              np.ascontiguousarray(dy, np.float32), None, None, o._ptr(dx), 1)
    return dx


def off_grid(po):
    """mask of dx elements no output pixel of a 1x1 / pad 0 layer reads: the data gradient is 0 there"""
    on_h = (np.arange(po.H) % po.sh == 0)
    on_w = (np.arange(po.W) % po.sw == 0)
    return ~(on_h[:, None] & on_w[None, :])


def bits(a):
    return np.ascontiguousarray(a).view(np.int32)


def setup(c, regime, math, sms):
    r = Run(c, math)
    q0, q1 = r.plans()
    assert regime(q0, q1, sms), f"the planners no longer produce this case's regime; forward {q0}, data gradient {q1}"
    return r, (q0, q1)


@pytest.mark.parametrize("cid,shape,regime,math,exact", CASES, ids=IDS)
def test_conv_float(rng, sms, cid, shape, regime, math, exact):
    r, plans = setup(shape(sms), regime, math, sms)
    po = r.po
    tol = 1e-3 if math == capi.MATH_TF32 else TOL
    x, w, b, dy = tensors(rng, po)
    W, B = dev(w), (dev(b) if b is not None else None)
    for op, a, want in ((capi.OP_FORWARD, x, oracle_y(po, x, w, b)), (capi.OP_BACKWARD_DATA, dy, oracle_dx(po, w, dy))):
        q = plans[op]
        what = f"{'forward' if op == capi.OP_FORWARD else 'data gradient'} on route {q['route']}"
        got = r.call(op, a, W, B)
        assert not np.isnan(got).any(), f"{what}: NaN in the output (an element never written, or NaN read from the workspace)"
        err = rel_err(got, want)
        assert err < tol, (what, err)
        if q["route"] == "gather_scatter":
            og = np.broadcast_to(off_grid(po), got.shape)
            assert (got[og] == 0).all(), f"{what}: off-grid elements of dx are not 0"
        again = r.call(op, a, W, B)
        assert np.array_equal(bits(got), bits(again)), f"{what}: not bit-identical run to run"
        if q["route"] not in TENSOR_CORE:
            continue
        # prepared filter cache, prefilled with NaN
        assert r.bind_cache(W)
        cached = r.call(op, a, W, B)
        assert np.array_equal(bits(got), bits(cached)), f"{what}: with the filter cache bound, not bit-identical"
        # 4 bytes off alignment: staged layers fall back to the gather kernel (which ignores the staged cache), gather layers
        # take the per-element epilogue
        un = r.call(op, a, W, B, off=1)
        assert not np.isnan(un).any(), f"{what}, unaligned: NaN in the output"
        assert rel_err(un, want) < tol, (what, "unaligned", rel_err(un, want))
        r.unbind_cache()
        if op == capi.OP_BACKWARD_DATA and q["route"] in STAGED:
            assert r.d.backward_data_accumulate_supported()
            dx0 = rng.standard_normal(po.x_shape()).astype(np.float32)
            acc = r.call(op, a, W, off=0, init=dx0, accumulate=True)
            assert np.array_equal(bits(acc), bits(dx0 + got)), f"{what}: accumulate is not dx0 + the data gradient bit for bit"


@pytest.mark.parametrize("cid,shape,regime,math,exact", [c for c in CASES if c[4]], ids=[c[0] for c in CASES if c[4]])
def test_conv_exact_integers(rng, sms, cid, shape, regime, math, exact):
    r, plans = setup(shape(sms), regime, math, sms)
    po = r.po

    def ints(shp):
        return rng.integers(-4, 5, shp).astype(np.float32)

    x, w, dy = ints(po.x_shape()), ints(po.w_shape()), ints(po.y_shape())
    b = ints((po.O,)) if po.has_bias else None
    W, B = dev(w), (dev(b) if b is not None else None)
    for op, a, want in ((capi.OP_FORWARD, x, oracle_y(po, x, w, b)), (capi.OP_BACKWARD_DATA, dy, oracle_dx(po, w, dy))):
        q = plans[op]
        assert np.abs(want).max() < 2 ** 24
        for off in ((0, 1) if q["route"] in TENSOR_CORE else (0,)):
            what = f"{'forward' if op == capi.OP_FORWARD else 'data gradient'} on route {q['route']}" + (", unaligned" if off else "")
            got = r.call(op, a, W, B, off=off)
            bad = np.argwhere(got != want)
            assert bad.size == 0, (f"{what}: {len(bad)} elements differ from the oracle, first at {tuple(bad[0])}: "
                                   f"got {got[tuple(bad[0])]}, want {want[tuple(bad[0])]}")

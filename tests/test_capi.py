"""CPU tests of the drop-in boundary: libb2c.so loads, exports every symbol include/b2c.h declares,
validates arguments like the reference's LayerSetUp CHECKs, and refuses to compute without a GPU."""
import ctypes as C
import os

import pytest

import caffe_mpi_b200 as m
from caffe_mpi_b200 import capi


def test_library_exports_every_declared_symbol():
    L = m.lib()
    syms = capi.declared_symbols()
    assert len(syms) >= 30
    missing = [s for s in syms if not hasattr(L, s)]
    assert not missing, missing
    assert b"sm_90a" in L.b2c_version()


def test_descriptor_validation_mirrors_layer_setup_checks():
    L = m.lib()
    h = C.c_void_p()
    bad = [
        m.ConvParams.make(1, 3, 8, 8, 4, 0),             # kernel 0: "Filter dimensions must be nonzero"
        m.ConvParams.make(1, 3, 8, 8, 4, 3, 0),          # stride 0
        m.ConvParams.make(1, 3, 8, 8, 4, 3, 1, 0, 1, 2),  # C % group
        m.ConvParams.make(1, 4, 8, 8, 3, 3, 1, 0, 1, 2),  # O % group
        m.ConvParams.make(1, 3, 2, 2, 4, 3),             # kernel larger than input
        m.ConvParams.make(1, 3, 8, 8, 4, 3, 1, -1),      # negative pad
    ]
    for p in bad:
        assert L.b2c_conv_desc_create(C.byref(p), 0, C.byref(h)) == -1
        assert len(L.b2c_last_error()) > 0
    assert L.b2c_conv_desc_create(C.byref(m.ConvParams.make(1, 3, 8, 8, 4, 3)), 7, C.byref(h)) == -1


def test_output_shape_and_workspace():
    # conv_layer.cpp:7-22 truncating division
    d = m.ConvDesc(m.ConvParams.make(2, 3, 8, 9, 4, 3, 2), capi.ENGINE_CAFFE)
    ho, wo = C.c_int(), C.c_int()
    assert m.lib().b2c_conv_out_shape(d._h, C.byref(ho), C.byref(wo)) == 0
    assert (ho.value, wo.value) == (3, 4)
    # CAFFE engine: one image's col buffer [Kd*G, Ho, Wo] floats; 1x1/s1/p0 needs none
    assert d.workspace_bytes(capi.OP_FORWARD) == 4 * 27 * 3 * 4
    d1 = m.ConvDesc(m.ConvParams.make(2, 3, 8, 9, 4, 1), capi.ENGINE_CAFFE)
    assert d1.workspace_bytes(capi.OP_FORWARD) == 0


def test_wgrad_plan_routes():
    """b2c_debug_wgrad_plan is host-only: the route choice of b2c_conv_backward_filter, with or without a device"""
    def plan(N, Cin, H, W, O, k, s=1, p=0, d=1, G=1, engine=capi.ENGINE_DEFAULT, math=None, algo=None):
        return m.ConvDesc(m.ConvParams.make(N, Cin, H, W, O, k, s, p, d, G, False), engine, math, algo).wgrad_plan()
    assert plan(8, 16, 16, 16, 32, 3, p=1)["route"] == "staged_3x3"
    assert plan(8, 16, 7, 7, 32, 3, p=1)["route"] == "staged_3x3_plane"
    assert plan(8, 16, 7, 7, 32, 1)["route"] == "staged_1x1_plane"
    assert plan(8, 16, 8, 8, 32, 1)["route"] == "staged_1x1"
    assert plan(8, 16, 6, 6, 32, 1)["route"] == "tma_1x1"
    assert plan(8, 16, 16, 16, 32, 1, s=2)["route"] == "compact_staged"
    assert plan(8, 16, 12, 12, 136, 1, s=2)["route"] == "compact_tma"
    assert plan(8, 16, 12, 12, 96, 1, s=2)["route"] == "gather"
    assert plan(8, 18, 7, 7, 32, 3, p=1)["route"] == "gather"                       # plane mode needs C % 4 == 0
    assert plan(8, 16, 16, 16, 32, 3, p=1, math=capi.MATH_TF32)["route"] == "gather"
    assert plan(8, 16, 16, 16, 32, 3, p=1, algo=capi.ALGO_SIMT)["route"] == "simt"
    assert plan(8, 16, 16, 16, 32, 3, p=1, engine=capi.ENGINE_CAFFE)["route"] == "caffe"
    q = plan(8, 16, 16, 16, 32, 3, p=1)
    assert (q["cols"], q["bpi"], q["nkb"]) == (72, 4, 32) and q["per"] * (q["splits"] - 1) < q["nkb"] <= q["per"] * q["splits"]
    d = m.ConvDesc(m.ConvParams.make(1, 3, 8, 8, 4, 3))
    assert m.lib().b2c_debug_wgrad_plan(d._h, (C.c_int * 5)(), 5) == -1


def test_conv_plan_routes():
    """b2c_debug_conv_plan is host-only: the route and tile plan of b2c_conv_forward (op 0) and b2c_conv_backward_data (op 1).
    The plans are asked for in a subprocess with the device hidden, so grids follow sm_count()'s no-device value of 132."""
    script = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
import caffe_mpi_b200 as m
from caffe_mpi_b200 import capi
def plan(N, Cin, H, W, O, k, s=1, p=None, d=1, G=1, engine=capi.ENGINE_DEFAULT, math=None, algo=None):
    kk = k if isinstance(k, int) else k
    p = (kk // 2 if isinstance(kk, int) else (kk[0] // 2, kk[1] // 2)) if p is None else p
    dd = m.ConvDesc(m.ConvParams.make(N, Cin, H, W, O, k, s, p, d, G, False), engine, math, algo)
    return [dd.conv_plan(0), dd.conv_plan(1)]
S = [
    plan(3, 32, 8, 16, 128, 1), plan(3, 32, 12, 15, 32, 3), plan(3, 32, 12, 16, 96, 3), plan(3, 32, 4, 63, 32, 3),
    plan(3, 32, 4, 64, 32, 3), plan(2, 32, 8, 16, 32, 5), plan(2, 32, 8, 16, 32, 7), plan(3, 48, 8, 16, 64, 3),
    plan(3, 32, 8, 16, 31, 3), plan(3, 32, 8, 16, 32, 3), plan(9, 32, 7, 7, 72, 3), plan(3, 32, 11, 13, 32, 3),
    plan(2, 3, 23, 23, 32, 7, s=2, p=3), plan(1, 512, 5, 5, 32, 3, s=2, p=1), plan(1, 516, 5, 5, 32, 3, s=2, p=1),
    plan(1, 127, 5, 5, 32, 3, s=2, p=1), plan(1, 129, 5, 5, 32, 3, s=2, p=1), plan(1, 8, 4, 4, 1024, 3, G=2),
    plan(1, 8, 4, 4, 1032, 3, G=2), plan(2, 32, 13, 13, 64, 1, s=2, p=0), plan(16, 64, 56, 56, 256, 3, s=2, p=1),
    plan(2, 32, 8, 16, 32, 3, math=capi.MATH_TF32), plan(2, 32, 8, 16, 32, 3, math=capi.MATH_FP32_3XTF32),
    plan(2, 32, 8, 16, 32, 3, algo=capi.ALGO_SIMT), plan(2, 32, 8, 16, 32, 3, engine=capi.ENGINE_CAFFE),
]
d = m.ConvDesc(m.ConvParams.make(1, 3, 8, 8, 4, 3))
L = m.lib()
import ctypes as C
refused = [L.b2c_debug_conv_plan(d._h, 0, (C.c_int * 7)(), 7), L.b2c_debug_conv_plan(d._h, 2, (C.c_int * 8)(), 8)]
print(json.dumps([S, refused]))
"""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    for k in ("B2C_NTILE", "B2C_CONV_STAGED", "B2C_CONV_STAGED_PLANE"):
        env.pop(k, None)
    out = subprocess.run([sys.executable, "-c", script, root], env=env, capture_output=True, text=True, check=True).stdout
    S, refused = json.loads(out.strip().splitlines()[-1])
    assert refused == [-1, -1]                                        # n < 8, and the weight gradient (b2c_debug_wgrad_plan's)

    def R(q, route, **want):
        return q["route"] == route and all(q[k] == v for k, v in want.items())
    (f, b), it = S[0], iter(S[1:])
    # one shape per route
    assert R(f, "staged", n_tile=128, m_tiles=3, n_tiles=1, tiles=3, grid=3, nkb=1, variant=128)      # 1x1 on 8x16: BWT 128
    assert R(b, "staged", n_tile=32, variant=128, nkb=2)
    f, b = next(it)
    assert R(f, "staged", variant=160) and R(b, "staged", variant=160)                                    # need == 160
    f, b = next(it)
    assert R(f, "staged", variant=192, n_tile=128) and R(b, "staged", variant=192, n_tile=32)             # need 165
    f, b = next(it)
    assert R(f, "staged", variant=256, m_tiles=6) and R(b, "staged", variant=256)                         # need == 256
    f, b = next(it)
    assert R(f, "gather", variant=1) and R(b, "gather", variant=1)                                        # need 261
    f, b = next(it)
    assert R(f, "staged", variant=256, nkb=13) and R(b, "staged")                                         # 25 taps
    f, b = next(it)
    assert R(f, "gather", variant=1, nkb=49) and R(b, "gather", variant=1)                                # 49 taps
    f, b = next(it)
    assert R(f, "gather", n_tile=64, variant=1) and R(b, "staged", n_tile=64, variant=192)                # C = 48
    f, b = next(it)
    assert R(f, "gather", n_tile=32) and R(b, "gather", variant=0)                                        # Cout 31 / 32
    f, b = next(it)
    assert R(f, "staged", n_tile=32) and R(b, "staged", n_tile=32)
    f, b = next(it)
    assert R(f, "staged_plane", variant=49, n_tile=128, m_tiles=4) and R(b, "gather", variant=1)          # 7x7: plane mode
    f, b = next(it)
    assert R(f, "gather") and R(b, "gather")                                                              # H*W % 4 != 0
    f, b = next(it)
    assert R(f, "gather", n_tile=32, variant=0, nkb=5, m_tiles=3) and R(b, "simt", n_tile=0, tiles=0, grid=0, variant=0)
    f, b = next(it)
    assert R(f, "gather", variant=1, nkb=144)                                                             # table: 1152 chunks
    f, b = next(it)
    assert R(f, "simt")
    f, b = next(it)
    assert R(f, "gather", variant=0, nkb=36)                                                              # table: 1152 elements
    f, b = next(it)
    assert R(f, "simt")
    f, b = next(it)
    assert R(f, "gather") and R(b, "gather", variant=1, nkb=144, tiles=2)                                 # dgrad table, G = 2
    f, b = next(it)
    assert R(f, "gather") and R(b, "simt")
    f, b = next(it)
    assert R(f, "gather") and R(b, "gather_scatter", n_tile=32, variant=1)
    f, b = next(it)
    assert R(f, "gather", n_tile=128, m_tiles=98, n_tiles=2, tiles=196, grid=132, nkb=18, variant=1)      # more than one wave
    for _ in range(2):                                                                                    # TF32, 3xTF32
        f, b = next(it)
        assert R(f, "gather") and R(b, "gather")
    f, b = next(it)
    assert R(f, "simt") and R(b, "simt")
    f, b = next(it)
    assert f == b == dict(route="caffe", n_tile=0, m_tiles=0, n_tiles=0, tiles=0, grid=0, nkb=0, variant=0)


def test_pool_plan_routes():
    """b2c_debug_pool_plan is host-only: the kernel b2c_pool_forward / b2c_pool_backward pick from the shape and the alignment of
    y, mask and dx (the routes test_layers_schedule_gpu.py runs), and the arguments PoolingLayer's CHECKs refuse"""
    A, OFF4, OFF8 = 1 << 20, (1 << 20) + 4, (1 << 20) + 8          # 16-byte aligned, 4 and 8 bytes past it

    def plan(d, NC, H, W, k, s, p, method=0, out=A, mask=A):
        q = capi.pool_plan(method, d, NC, H, W, (k, k) if isinstance(k, int) else k, (s, s) if isinstance(s, int) else s,
                           (p, p) if isinstance(p, int) else p, out, mask)
        return q["route"], q["Ho"], q["Wo"], (q["q"] if d == 0 else q["rpb"])
    # (NC, H, W, k, s, p): forward, backward
    table = [
        ((512, 112, 112, 3, 2, 0), ("max_window", 56, 56, 4), ("max_bwd_quad", 56, 56, 0)),
        ((24, 56, 56, 3, 2, 0), ("max_window", 28, 28, 4), ("max_bwd_quad", 28, 28, 0)),
        ((24, 28, 28, 3, 2, 0), ("max_window", 14, 14, 2), ("max_bwd_quad", 14, 14, 0)),
        ((24, 14, 14, 3, 2, 0), ("max_scalar", 7, 7, 0), ("max_bwd_row", 7, 7, 9)),
        ((24, 28, 28, 3, 1, 1), ("max_window", 28, 28, 4), ("max_bwd_quad", 28, 28, 0)),
        ((24, 14, 14, 3, 1, 1), ("max_window", 14, 14, 2), ("max_bwd_row", 14, 14, 9)),
        ((24, 7, 7, 3, 1, 1), ("max_scalar", 7, 7, 0), ("max_bwd_row", 7, 7, 18)),
        ((6144, 55, 55, 3, 2, 0), ("max_scalar", 27, 27, 0), ("max_bwd_row", 27, 27, 2)),
        ((24, 13, 13, 3, 2, 0), ("max_window", 6, 6, 2), ("max_bwd_row", 6, 6, 9)),
        ((4, 224, 224, 2, 2, 0), ("max_window", 112, 112, 4), ("max_bwd_quad", 112, 112, 0)),
        ((24, 14, 14, 2, 2, 0), ("max_scalar", 7, 7, 0), ("max_bwd_row", 7, 7, 9)),
        ((12, 30, 44, 3, 2, 0), ("max_window", 15, 22, 2), ("max_bwd_quad", 15, 22, 0)),
        ((12, 44, 30, 3, 2, 0), ("max_scalar", 22, 15, 0), ("max_bwd_row", 22, 15, 4)),
        ((12, 10, 16, 3, 2, 0), ("max_window", 5, 8, 4), ("max_bwd_quad", 5, 8, 0)),             # ceil mode: partial last window
        ((12, 15, 15, 3, 2, 1), ("max_window", 8, 8, 4), ("max_bwd_row", 8, 8, 8)),
        ((12, 8, 8, 3, 2, 1), ("max_scalar", 5, 5, 0), ("max_bwd_quad", 5, 5, 0)),
        ((12, 9, 9, 3, 2, 1), ("max_scalar", 5, 5, 0), ("max_bwd_row", 5, 5, 14)),
        ((12, 5, 130, 3, 1, 1), ("max_window", 5, 130, 2), ("max_bwd_row", 5, 130, 1)),
        ((12, 11, 13, (3, 2), (2, 1), (1, 0)), ("max_scalar", 6, 12, 0), ("max_bwd_row", 6, 12, 9)),
        ((12, 6, 3, 2, 2, 0), ("max_window", 3, 2, 2), ("max_bwd_row", 3, 2, 42)),
        ((300, 5, 1, 1, 1, 0), ("max_scalar", 5, 1, 0), ("max_bwd_row", 5, 1, 128)),
        ((12, 9, 9, 1, 2, 0), ("max_scalar", 5, 5, 0), ("max_bwd_row", 5, 5, 14)),
    ]
    for args, f, b in table:
        assert plan(0, *args) == f, (args, plan(0, *args))
        assert plan(1, *args) == b, (args, plan(1, *args))
    for args in ((24, 7, 7, 7, 1, 0), (24, 14, 14, 5, 3, 0), (24, 8, 8, 3, 2, 1), (24, 9, 9, 2, 2, 0), (24, 10, 14, (3, 2), (2, 3), (1, 0))):
        assert plan(0, *args, method=1)[0] == plan(1, *args, method=1)[0] == "ave"
    assert plan(0, 24, 10, 14, (3, 2), (2, 3), (1, 0), method=1) == ("ave", 6, 5, 0)
    # alignment: y and mask must both sit on 4Q bytes for the window kernel, dx on 16 for the quad kernel
    assert plan(0, 24, 56, 56, 3, 2, 0, out=OFF4)[0] == plan(0, 24, 56, 56, 3, 2, 0, mask=OFF4)[0] == "max_scalar"
    assert plan(0, 24, 56, 56, 3, 2, 0, out=OFF8)[0] == "max_scalar"
    assert plan(0, 24, 28, 28, 3, 2, 0, out=OFF8, mask=OFF8) == ("max_window", 14, 14, 2)
    assert plan(1, 24, 56, 56, 3, 2, 0, out=OFF8) == ("max_bwd_row", 28, 28, 2)
    # refused, by the query and by both entry points, before anything is launched
    L = m.lib()
    one = C.c_void_p(A)
    bad = [
        (0, 8, 8, 0, 3, 1, 1, 0, 0),          # kernel 0
        (0, 8, 8, 3, 0, 1, 1, 0, 0),
        (0, 8, 8, 3, 3, 0, 1, 0, 0),          # stride 0
        (0, 8, 8, 3, 3, 1, 0, 0, 0),
        (0, 8, 8, 3, 3, 1, 1, 3, 0),          # pad == kernel
        (0, 8, 8, 3, 3, 1, 1, 0, 3),
        (0, 8, 8, 3, 3, 1, 1, -1, 0),         # negative pad
        (0, 0, 8, 3, 3, 1, 1, 0, 0),          # empty map
        (0, 8, 0, 3, 3, 1, 1, 0, 0),
        (0, 1, 8, 3, 3, 1, 1, 0, 0),          # H + 2 pad < kernel: no output row
        (0, 8, 2, 5, 5, 1, 1, 1, 1),          # W + 2 pad < kernel
        (2, 8, 8, 3, 3, 1, 1, 0, 0),          # STOCHASTIC
    ]
    for method, H, W, kh, kw, sh, sw, ph, pw in bad:
        for d in (0, 1):
            with pytest.raises(capi.B2CError):
                capi.pool_plan(method, d, 4, H, W, (kh, kw), (sh, sw), (ph, pw), A, A)
        assert L.b2c_pool_forward(method, 4, H, W, kh, kw, sh, sw, ph, pw, one, one, one, None) == -1
        assert L.b2c_pool_backward(method, 4, H, W, kh, kw, sh, sw, ph, pw, one, one, one, None) == -1
    with pytest.raises(capi.B2CError):
        capi.pool_plan(0, 0, 0, 8, 8, (3, 3), (1, 1), (0, 0))              # no planes
    assert L.b2c_debug_pool_plan(0, 0, 4, 8, 8, 3, 3, 1, 1, 0, 0, one, one, (C.c_int * 4)(), 4) == -1     # n < 5


@pytest.mark.skipif(any(k.startswith("B2C_BN_") for k in os.environ), reason="the table is the default switches'")
def test_bn_plan_regimes():
    """b2c_debug_bn_plan is host-only: the launch every BatchNorm training entry point takes (the regimes test_bn_schedule_gpu.py
    runs), at 132 SMs (an H100 SXM, and the count without a device), and the shapes the entry points refuse"""
    A, OFF4 = 1 << 20, (1 << 20) + 4
    sms = 132
    try:
        import torch
        if torch.cuda.is_available():
            sms = torch.cuda.get_device_properties(0).multi_processor_count
    except Exception:
        pass
    if sms != 132:
        pytest.skip(f"the table is 132 SMs' ({sms} here)")

    def plan(d, form, N, Cc, H, W, ptr=A):
        q = capi.bn_plan(d, form, N, Cc, H * W, [ptr])
        return q["launches"], q["cs"], q["threads"], q["park"], q["prefetch"], q["vec"]
    # (N, C, H, W): forward fused, backward fused, backward fused_res -- (launches, cs, threads, park, prefetch, float4)
    table = [
        ((64, 64, 112, 112), (1, 8, 512, 0, 0, True), (1, 8, 512, 0, 0, True), (1, 8, 512, 0, 0, True)),     # bn_conv1: 392 KB slices
        ((64, 64, 56, 56), (1, 8, 512, 1, 1, True), (1, 8, 512, 1, 1, True), (1, 8, 512, 2, 1, True)),        # res2: 98 KB slices
        ((64, 256, 56, 56), (1, 8, 512, 1, 1, True), (1, 8, 512, 1, 1, True), (1, 8, 512, 2, 1, True)),
        ((64, 128, 28, 28), (1, 2, 512, 1, 1, True), (1, 2, 512, 1, 1, True), (1, 2, 512, 2, 1, True)),       # res3
        ((64, 512, 28, 28), (1, 2, 512, 1, 1, True), (1, 2, 512, 1, 1, True), (1, 2, 512, 2, 1, True)),
        ((64, 256, 14, 14), (1, 1, 256, 1, 1, True), (1, 1, 512, 3, 1, True), (1, 1, 512, 3, 1, True)),       # res4: 256-thread forward
        ((64, 1024, 14, 14), (1, 1, 256, 1, 1, True), (1, 1, 512, 3, 1, True), (1, 1, 512, 3, 1, True)),
        ((64, 512, 7, 7), (1, 1, 128, 1, 1, False), (1, 1, 128, 3, 1, False), (1, 1, 128, 3, 1, False)),     # res5: S = 49, scalar
        ((64, 2048, 7, 7), (1, 1, 128, 1, 1, False), (1, 1, 128, 3, 1, False), (1, 1, 128, 3, 1, False)),
        ((64, 40, 35, 35), (1, 4, 512, 1, 1, False), (1, 4, 512, 1, 1, False), (1, 4, 512, 2, 1, False)),     # scalar, 512 threads, cs 4
        ((37, 70, 30, 30), (1, 2, 512, 1, 1, True), (1, 2, 512, 1, 1, True), (1, 2, 512, 2, 1, True)),        # slices end mid-plane
    ]
    for shape, f, b, r in table:
        assert plan(0, "fused", *shape) == plan(0, "fused_res", *shape) == f, (shape, plan(0, "fused", *shape))
        assert plan(1, "fused", *shape) == b, (shape, plan(1, "fused", *shape))
        assert plan(1, "fused_res", *shape) == r, (shape, plan(1, "fused_res", *shape))
        for d, one in ((0, f), (1, b)):          # the unfused layers: the same reduction geometry, two launches, nothing parked
            assert plan(d, "unfused", *shape) == (2, one[1], one[2], 0, 0, one[5]), (shape, d)
    # one pointer 4 bytes off 16-byte alignment takes every form to one float at a time; null pointers do not count
    for d in (0, 1):
        for form in capi.BN_FORMS:
            assert plan(d, form, 64, 256, 14, 14, OFF4)[5] is False
            assert capi.bn_plan(d, form, 64, 256, 196, [A, None, A])["vec"] is True
    # refused, by the query and by the entry points, before anything is launched
    L = m.lib()
    one = C.c_void_p(A)
    for N, Cc, S in ((0, 4, 4), (4, 0, 4), (4, 4, 0), (-1, 4, 4), (4, 65536, 4), (1 << 16, 4, 1 << 15)):
        for d in (0, 1):
            for form in capi.BN_FORMS:
                with pytest.raises(capi.B2CError, match="channel extent out of range"):
                    capi.bn_plan(d, form, N, Cc, S, [A])
        assert L.b2c_bn_forward_train(N, Cc, S, one, None, None, 1e-5, 0.9, 1, one, one, one, one, one, one, None) == -1
        assert L.b2c_bn_backward(N, Cc, S, one, one, None, one, one, one, one, None) == -1
        assert L.b2c_bn_forward_train_fused(N, Cc, S, one, None, None, 1e-5, 0.9, 1, one, one, one, one, one, 0, None) == -1
        assert L.b2c_bn_backward_fused(N, Cc, S, one, one, one, one, None, None, one, one, one, 0, None) == -1
        assert L.b2c_bn_forward_train_fused_res(N, Cc, S, one, None, None, 1e-5, 0.9, 1, one, one, one, one, one, one, 1, None) == -1
        assert L.b2c_bn_backward_fused_res(N, Cc, S, one, None, one, one, one, one, None, None, one, one, one, None, None) == -1
    out = (C.c_int * 6)()
    ptrs = (C.c_void_p * 1)(A)
    assert L.b2c_debug_bn_plan(2, 0, 4, 4, 4, ptrs, 1, out, 6) == -1                  # dir
    assert L.b2c_debug_bn_plan(0, 3, 4, 4, 4, ptrs, 1, out, 6) == -1                  # form
    assert L.b2c_debug_bn_plan(0, 0, 4, 4, 4, ptrs, 7, out, 6) == -1                  # more than 6 pointers
    assert L.b2c_debug_bn_plan(0, 0, 4, 4, 4, ptrs, 1, out, 5) == -1                  # n < 6


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    L = m.lib()
    d = m.ConvDesc(m.ConvParams.make(1, 3, 8, 8, 4, 3))
    one = C.c_void_p(16)
    rc = L.b2c_conv_forward(d._h, one, one, one, one, None, 0, None)
    assert rc == -2 and b"no CPU fallback" in L.b2c_last_error()
    assert L.b2c_sgemm(0, 0, 2, 2, 2, 1.0, one, one, 0.0, one, None) == -2

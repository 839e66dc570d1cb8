"""CPU tests of the drop-in boundary: libb2c.so loads, exports every symbol include/b2c.h declares,
validates arguments like the reference's LayerSetUp CHECKs, and refuses to compute without a GPU."""
import ctypes as C

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
